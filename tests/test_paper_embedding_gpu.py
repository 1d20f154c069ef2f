"""GPU tests of the DALL-E paper's input embedding: row / column image positions (image_position_embedding "row_col")
and a padding token per text position (per_position_padding).

Kernels
  * db200_pos_compose: bit-exact against the bf16-rounded definition bf16_rn(float(row[r]) + float(col[c])).
  * db200_pos_fold: against float64.  Every output element is g + x_1 + ... + x_n (n = 1 for a text row, W for a grid
    row or column) summed in fp32 in a fixed order, n additions of n + 1 terms.  Recursive summation bounds the error
    of that by gamma_n * sum |terms|, gamma_n = n u / (1 - n u), u = 2^-24 (Higham, Accuracy and Stability of Numerical
    Algorithms, 2nd ed., eq. 4.4), which is the bound asserted.  Two runs are bit-identical.
  * db200_assemble_tokens_pp: bit-exact against oracle/dalle_input.py, pads at random positions and at row ends, with
    and without caption dropout, with and without image codes.
Engine against the oracle: loss, logits and every gradient at the full dalle_example shape and the dalle_coco
geometry, with the bounds of tests/test_parity_baseline_gpu.py; again with the three dropout rates at 0.1 and with a
[axial_row, conv, global] schedule.  Each mutated oracle (oracle/dalle_input.py MUTATIONS) fails those bounds.
Also: a bitwise-reproducible step, generation (greedy decode, graph replay, prefill, guided and image-prefixed
completion), save / resume through dalle_model_fn and the cross-scheme load error, ZeRO-1 on one GPU against the
replicated step bitwise, W in-process ranks against one rank with W micro-batches bitwise, generate_dalle.py end to
end, and, without the keys, the engine's kernel sequence.
"""
import json
import os

import numpy as np
import pytest
import torch

import conv_oracle as OC
from test_data_parallel_gpu import _check_coverage, _dalle_data, _dalle_params, _dalle_ranks, _dalle_reference, \
    _seq_len, rec  # noqa: F401  (rec is a fixture)
from test_parity_baseline_gpu import _randomise_small_params, record, relfro
from test_zero1_gpu import Loopback, _twin_from, assert_same_bits

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
U = 2.0 ** -24


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def _gamma(n):
    return n * U / (1 - n * U)


# ================================================================================================== kernels
@pytest.mark.parametrize("TL,W,d", [(256, 32, 512), (256, 32, 1024), (256, 32, 4096), (0, 8, 256), (5, 3, 8)])
def test_pos_compose_is_the_bf16_rounded_definition(ops, TL, W, d):
    g = torch.Generator(device=DEV).manual_seed(TL + W + d)
    wpe = (torch.randn(TL, d, generator=g, device=DEV) * 0.01).to(BF16)
    row = (torch.randn(W, d, generator=g, device=DEV) * 0.01).to(BF16)
    col = (torch.randn(W, d, generator=g, device=DEV) * 0.01).to(BF16)
    col[0, :4] = -row[0, :4]                               # exact cancellation: +0
    row[1, :4] = torch.tensor([65280.0, -65280.0, 3e38, 1e-40], dtype=BF16)   # overflow to inf, subnormal
    col[1, :4] = torch.tensor([65280.0, -65280.0, 3e38, 1e-40], dtype=BF16)
    out = torch.full((TL + W * W, d), float("nan"), dtype=BF16, device=DEV)
    ops.pos_compose(wpe, row, col, out)
    r = torch.arange(W, device=DEV).repeat_interleave(W)
    c = torch.arange(W, device=DEV).repeat(W)
    want = torch.cat([wpe, (row.float()[r] + col.float()[c]).to(BF16)])
    assert_same_bits(out.view(-1), want.view(-1), "pos_compose")


@pytest.mark.parametrize("TL,W,d", [(256, 32, 512), (256, 32, 1024), (256, 32, 4096), (0, 8, 256), (5, 3, 8)])
def test_pos_fold_against_float64_and_reproducible(ops, TL, W, d):
    g = torch.Generator(device=DEV).manual_seed(7 * W + d)
    dpos = torch.randn(TL + W * W, d, generator=g, device=DEV) * torch.rand(TL + W * W, 1, generator=g, device=DEV)
    g0 = [torch.randn(n, d, generator=g, device=DEV) for n in (TL, W, W)]
    outs = []
    for _ in range(2):
        o = [t.clone() for t in g0]
        ops.pos_fold(dpos, *o)
        outs.append(o)
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert_same_bits(a.view(-1), b.view(-1), "pos_fold: two runs")
    x = dpos.double()
    img = x[TL:].view(W, W, d)
    exact = [g0[0].double() + x[:TL], g0[1].double() + img.sum(1), g0[2].double() + img.sum(0)]
    absum = [g0[0].double().abs() + x[:TL].abs(), g0[1].double().abs() + img.abs().sum(1),
             g0[2].double().abs() + img.abs().sum(0)]
    worst = 0.0
    for name, got, ex, ab, n in zip(("wpe", "row", "col"), outs[0], exact, absum, (1, W, W)):
        if got.numel() == 0:
            continue
        err = (got.double() - ex).abs()
        bound = _gamma(n) * ab
        assert (err <= bound).all(), (name, float((err - bound).max()))
        worst = max(worst, float((err / bound.clamp_min(1e-300)).max()))
    record(f"pos_fold TL={TL} W={W} d={d}", worst_error_over_bound=worst)


def test_assemble_tokens_pp_matches_the_oracle(ops):
    from dalle_mtf_b200 import lib as L
    from oracle import dalle_input as I
    from oracle import dalle_local as OL
    TL, isl, tv, iv, pad = 256, 1024, 50258, 512, 50257
    cfg = OL.LocalConfig(512, 1, 4, tv, iv, TL, isl)
    inp = I.InputConfig("row_col", True, pad)
    B = 37
    g = torch.Generator().manual_seed(3)
    text = torch.randint(0, tv, (B, TL), generator=g)
    text[torch.rand(B, TL, generator=g) < 0.1] = pad                  # pads at random positions
    for b in range(B):
        text[b, int(torch.randint(1, TL + 1, (1,), generator=g)):] = pad   # and at row ends (some rows have none)
    text[0] = pad
    img = torch.randint(0, iv, (B, isl), generator=g)
    t_d, i_d = text.to(I32).to(DEV), img.to(I32).to(DEV)
    off = tv + TL
    out = torch.empty(B, TL + isl, dtype=I32, device=DEV)
    ops.assemble_tokens_pp(t_d, i_d, out, off, pad, tv)
    assert torch.equal(out.cpu().long(), I.assemble(text, img, cfg, inp))
    for rate, seed, step, row0 in ((0.3, 5, 2, 0), (0.5, 9, 11, 1000)):
        drop = L.make_dropout(rate, seed, step, L.SITE_CAPTION, row0)
        ops.assemble_tokens_pp(t_d, i_d, out, off, pad, tv, caption_drop=drop)
        want = I.assemble(text, img, cfg, inp, caption_drop=(rate, seed, step, row0))
        assert torch.equal(out.cpu().long(), want)
        assert (want[1:, :TL] == tv + torch.arange(TL)).all(1).any()     # some caption was dropped
    caps = torch.empty(B, TL, dtype=I32, device=DEV)                    # captions alone (the sampler's use)
    ops.assemble_tokens_pp(t_d, None, caps, 0, pad, tv)
    assert torch.equal(caps.cpu().long(), I.map_pads(text, cfg, inp))
    with pytest.raises(L.DB200Error):
        ops.assemble_tokens_pp(t_d, i_d, out, off, -1, tv)


# ================================================================================================== engine parity
def _engine_vs_oracle(d, L, H, tv, iv, ts, isl, B, recompute, seed, types=None, rates=None, kernel=5, inp=None,
                      mutations=()):
    """(violations of the true oracle, {mutation: violations}) of one engine step against oracle/dalle_input.py.
    Violations name the bounds of tests/test_parity_baseline_gpu.py that fail."""
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle_input as I
    from oracle import dalle_local as OL
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    inp = inp or I.InputConfig("row_col", True, tv - 1)
    if types is not None and set(types) & {"axial_row", "axial_col", "conv"}:
        cfg = OC.ConvConfig(d, L, H, tv, iv, ts, isl, attention_types=tuple(types), conv_attention_kernel=kernel)
        base = OC.forward
    else:
        cfg = OL.LocalConfig(d, L, H, tv, iv, ts, isl, attention_types=None if types is None else tuple(types))
        base = OL.forward
    params = I.init_params(cfg, inp, seed)
    g = torch.Generator().manual_seed(seed + 1)
    _randomise_small_params(params, g)
    text = torch.randint(0, tv - 1, (B, ts), generator=g)
    for b in range(B):
        text[b, 5 + 20 * b:] = tv - 1
    text[:, 2] = tv - 1                                          # a pad inside the caption too
    img = torch.randint(0, iv, (B, isl), generator=g)
    step = 3 if rates else None
    dropout = ((rates,) * 3, seed, step, 0) if rates else None

    eng = DalleEngine(d, L, H, tv, iv, ts, isl, recompute_grad=recompute, attention_types=types,
                      conv_attention_kernel=kernel, dropout=(rates or 0.0,) * 3, dropout_seed=seed,
                      image_position_embedding=inp.image_position_embedding,
                      per_position_padding=inp.per_position_padding)
    eng.load_params(params)
    tok = torch.empty(B, ts + isl, dtype=I32, device=DEV)
    if inp.per_position_padding:
        from dalle_mtf_b200 import ops
        ops.assemble_tokens_pp(text.to(I32).to(DEV), img.to(I32).to(DEV), tok, eng.image_offset, inp.padding_id,
                                eng.pad_base)
    else:
        tok.copy_(I.assemble(text, img, cfg, inp))
    T = tok.numel()
    eng.zero_grads()
    acc = eng.forward(tok, step=step)
    eng.backward(1.0 / T)
    torch.cuda.synchronize()
    loss = acc.item() / T
    rows = eng._bufs["loss_rows"].float().cpu().view(B, -1)
    lg = eng.logits(tok).float().cpu() if rates is None else None
    grads = eng.export_params(eng.grads)
    assert (eng.G("wout")[:, eng.V:] == 0).all() and (eng.G("bout")[eng.V:] == 0).all()
    n_params = eng.n_params()
    del eng
    torch.cuda.empty_cache()
    assert n_params == sum(v.numel() for v in params.values())

    def violations(mutate):
        tokens = I.assemble(text, img, cfg, inp, mutate=mutate)
        loss32, rows32, logits32, g32 = I.loss_and_grads(params, tokens, cfg, inp, dropout, False, mutate=mutate,
                                                         base=base)
        _, _, logits16, g16 = I.loss_and_grads(params, tokens, cfg, inp, dropout, True, mutate=mutate, base=base)
        bad = []
        loss_rel = abs(loss - loss32.item()) / loss32.item()
        if loss_rel > 1e-3:
            bad.append(("loss", loss_rel))
        rows_err = relfro(rows, rows32)
        if rows_err > 5e-3:
            bad.append(("loss_rows", rows_err))
        e_eng = e_ref = None
        if lg is not None:
            e_eng, e_ref = relfro(lg, logits32), relfro(logits16, logits32)
            if not (e_eng <= 1.25 * e_ref + 2e-3 and e_eng <= 2e-2):
                bad.append(("logits", e_eng, e_ref))
        worst = (None, 0.0)
        assert set(g32) == set(grads)
        for k in g32:
            ee, er = relfro(grads[k], g32[k]), relfro(g16[k], g32[k])
            if ee > 1.25 * er + 1e-2:
                bad.append(("grad " + k, ee, er))
            if ee / (1.25 * er + 1e-2) > worst[1]:
                worst = (k, ee / (1.25 * er + 1e-2))
        record(f"paper-input {mutate or 'oracle'}", loss_rel=loss_rel, rows_relfro=rows_err, logits_engine=e_eng,
               logits_refbf16=e_ref, closest_grad=worst[0], its_share_of_bound=worst[1], violations=len(bad))
        return bad

    return violations(None), {m: violations(m) for m in mutations}


def test_dalle_example_shape_matches_oracle():
    """EX: d512 / L6 / H4 / S = 256 + 32^2 / V = 50 258 + 256 + 512 + 1, B = 2, both keys."""
    bad, _ = _engine_vs_oracle(512, 6, 4, 50258, 512, 256, 1024, 2, False, seed=11)
    assert not bad, bad


def test_dalle_coco_geometry_recompute_matches_oracle():
    """CO geometry: d1024 / H16 (dh 64) / S1280 / recompute_grad, L cut to 2, B = 1, both keys."""
    bad, _ = _engine_vs_oracle(1024, 2, 16, 50258, 8192, 256, 1024, 1, True, seed=12)
    assert not bad, bad


def test_dalle_example_with_dropout_matches_oracle():
    """EX with embed, attention and residual dropout at 0.1 (masks of a training step), L cut to 2."""
    bad, _ = _engine_vs_oracle(512, 2, 4, 50258, 512, 256, 1024, 2, False, seed=13, rates=0.1)
    assert not bad, bad


def test_mixed_sparse_schedule_matches_oracle():
    """EX width with [axial_row, conv, global] layers (conv k = 5) against tests/conv_oracle.py."""
    bad, _ = _engine_vs_oracle(512, 3, 4, 50258, 512, 256, 1024, 1, False, seed=14,
                               types=["axial_row", "conv", "global"])
    assert not bad, bad


def test_each_mutated_oracle_fails_and_each_key_alone_matches():
    from oracle import dalle_input as I
    bad, mut = _engine_vs_oracle(256, 2, 2, 300, 64, 24, 64, 3, False, seed=15, mutations=I.MUTATIONS)
    assert not bad, bad
    for m, v in mut.items():
        assert v, f"the oracle mutated by {m!r} still matches the engine"
    for inp in (I.InputConfig("row_col", False, None), I.InputConfig("absolute", True, 299)):
        bad, _ = _engine_vs_oracle(256, 2, 2, 300, 64, 24, 64, 3, False, seed=16, inp=inp)
        assert not bad, (inp, bad)


# ================================================================================================== step, layout
def _small_engine(**kw):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    args = dict(image_position_embedding="row_col", per_position_padding=True)
    args.update(kw)
    return DalleEngine(256, 2, 2, 300, 64, 24, 64, **args)


def test_training_step_is_bitwise_reproducible():
    outs = []
    for _ in range(2):
        eng = _small_engine(dropout=(0.1, 0.1, 0.1), dropout_seed=4)
        eng.init_params(seed=2)
        g = torch.Generator(device=DEV).manual_seed(1)
        tok = torch.randint(0, eng.V - 1, (4, eng.S), generator=g, device=DEV, dtype=I32)
        for step in range(2):
            eng.zero_grads()
            for mb in range(2):
                eng.forward(tok[2 * mb:2 * mb + 2], step=step, row0=2 * mb, global_batch=4)
                eng.backward(1.0 / tok.numel())
            grads = eng.grads.clone()
            eng.optimizer_step(1e-3, weight_decay=0.01)
        torch.cuda.synchronize()
        outs.append((grads, eng.master.clone(), eng.shadow.clone(), eng.pos_table.clone()))
    for a, b, what in zip(*outs, ("gradients", "master", "bf16 parameters", "position table")):
        assert_same_bits(a.view(-1), b.view(-1), what)
    # the position table is the composition of the bf16 parameters after the step
    eng2 = _small_engine()
    eng2.shadow.copy_(outs[0][2])
    eng2._compose_pos()
    assert_same_bits(eng2.pos_table.view(-1), outs[0][3].view(-1), "position table after optimizer_step")


def test_layout_vocabulary_and_bucket_of_the_engine():
    from dalle_mtf_b200.dalle_engine import param_layout
    eng = _small_engine()
    assert (eng.V, eng.image_offset, eng.pad_base, eng.grid_w) == (300 + 24 + 64 + 1, 324, 300, 8)
    assert eng.layout.entries == param_layout(256, 2, eng.V, eng.S, 24, 8).entries
    assert set(eng.export_params()) == set(eng.export_params(eng.grads))
    seen = []
    eng.init_params(0)
    tok = torch.randint(0, eng.V - 1, (1, eng.S), device=DEV, dtype=I32)
    eng.zero_grads()
    eng.forward(tok)
    eng.backward(1.0, on_bucket_ready=lambda s, e: seen.append((s, e)))
    assert seen[-1] == eng.layout.span("wte", "image_col") == (0, eng.layout.entries["l0.ln1_g"][0])
    plain = _small_engine(image_position_embedding=None, per_position_padding=None)
    assert plain.layout.entries == param_layout(256, 2, 300 + 64 + 1, 88).entries
    assert set(plain.export_params()) == {k for k in eng.export_params() if "image_" not in k}
    segs = eng._decay_segments()
    s, e = eng.layout.span("wte", "image_col")
    assert any(a <= s and e <= b and dec for a, b, dec in segs)       # the new matrices decay like wpe


def _op_sequence(monkeypatch, eng, tok, step=None):
    """Ordered names of the ops.* calls of one forward + backward + optimizer_step."""
    from dalle_mtf_b200 import ops
    seq = []
    for name in [n for n in dir(ops) if not n.startswith("_") and callable(getattr(ops, n))]:
        fn = getattr(ops, name)
        if getattr(fn, "__module__", None) != ops.__name__:
            continue

        def wrap(*a, _fn=fn, _n=name, **k):
            seq.append(_n)
            return _fn(*a, **k)
        monkeypatch.setattr(ops, name, wrap)
    eng.zero_grads()
    eng.forward(tok, step=step)
    eng.backward(1.0)
    eng.optimizer_step(1e-3)
    monkeypatch.undo()
    return seq


def test_without_the_keys_the_kernel_sequence_is_unchanged(monkeypatch):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    tok = torch.randint(0, 300, (2, 88), device=DEV, dtype=I32)
    for kw in ({}, {"dropout": (0.1, 0.1, 0.1)}):
        a = DalleEngine(256, 2, 2, 300, 64, 24, 64, **kw)
        b = DalleEngine(256, 2, 2, 300, 64, 24, 64, image_position_embedding="absolute", per_position_padding=False,
                        **kw)
        a.init_params(1); b.init_params(1)
        sa = _op_sequence(monkeypatch, a, tok, step=0)
        sb = _op_sequence(monkeypatch, b, tok, step=0)
        assert sa == sb and not {"pos_compose", "pos_fold", "assemble_tokens_pp"} & set(sa)
        c = DalleEngine(256, 2, 2, 300, 64, 24, 64, image_position_embedding="row_col", **kw)
        c.init_params(1)
        sc = _op_sequence(monkeypatch, c, tok, step=0)
        # row / column positions add exactly the fold after the embedding backward and the compose after the step
        i = sa.index("embed_bwd")
        assert sc == sa[:i + 1] + ["pos_fold"] + sa[i + 1:] + ["pos_compose"]


# ================================================================================================== generation
def _sharp_engine_and_text(B=3, tv=300, iv=64, ts=10, isl=16):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle_input as I
    from oracle import dalle_local as OL
    cfg = OL.LocalConfig(256, 2, 2, tv, iv, ts, isl)
    inp = I.InputConfig("row_col", True, 7)
    params = I.init_params(cfg, inp, 3)
    g = torch.Generator().manual_seed(9)
    for k in params:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if "wte" in k or "wout" in k or k.endswith("kernel") or "positional" in k:
            params[k] = params[k] * 4
    eng = DalleEngine(256, 2, 2, tv, iv, ts, isl, image_position_embedding="row_col", per_position_padding=True)
    eng.load_params(params)
    text = torch.randint(0, tv, (B, ts), generator=g)
    text[0, 4:] = 7
    text[1, 1] = 7
    return eng, text.to(I32).to(DEV), cfg, inp


def test_greedy_decode_graph_replay_and_prefill():
    from dalle_mtf_b200.sampling import DalleSampler
    from oracle import dalle_input as I
    eng, text, cfg, inp = _sharp_engine_and_text()
    ts, S, off, iv = eng.text_seq_len, eng.S, eng.image_offset, eng.image_vocab_size
    smp = DalleSampler(eng, padding_id=7)
    toks, step_logits = smp.generate(text, temperature=0, return_logits=True)
    torch.cuda.synchronize()
    assert torch.equal(toks[:, :ts].cpu().long(), I.map_pads(text.cpu(), cfg, inp))     # the training mapping
    img = toks[:, ts:]
    assert (img >= off).all() and (img < off + iv).all()
    full = eng.logits(toks)
    dec = torch.stack(step_logits, 1)
    assert relfro(dec, full[:, :S - 1]) < 2e-2
    rng = full[:, ts - 1:S - 1, off:off + iv]
    top2 = rng.topk(2, -1).values
    clear = (top2[..., 0] - top2[..., 1]) > 0.05 * rng.abs().max()
    same = (rng.argmax(-1) + off) == img
    assert (same | ~clear).all() and clear.float().mean() > 0.2 and same.float().mean() > 0.8
    # graph replay = eager
    assert torch.equal(smp.generate_graphed(text, temperature=0.0), toks)
    # prefill of the first P positions: the logits of position P - 1, within the decode tests' bound
    P = ts + 5
    kc = [torch.zeros(3, S, eng.H, eng.dh, dtype=BF16, device=DEV) for _ in range(eng.L)]
    vc = [torch.zeros_like(c) for c in kc]
    pl = eng.prefill(toks[:, :P].contiguous(), kc, vc)
    assert relfro(pl[:, :eng.V], full[:, P - 1]) < 2e-2
    assert relfro(pl[:, :eng.V], dec[:, P - 1]) < 2e-2


def test_guided_and_image_prefixed_completion_use_per_position_pads():
    from dalle_mtf_b200.sampling import DalleSampler
    eng, text, cfg, inp = _sharp_engine_and_text()
    ts, off, iv, B = eng.text_seq_len, eng.image_offset, eng.image_vocab_size, 3
    pads = torch.arange(ts, device=DEV, dtype=I32) + eng.pad_base
    smp = DalleSampler(eng, padding_id=7)
    prefix = torch.randint(0, iv, (B, 4), device=DEV, dtype=I32)
    torch.manual_seed(0)
    out = smp.complete(text, prefix, samples_per_prompt=2, temperature=1.0, top_k=8, guidance_scale=3.0)
    R = 2 * B
    assert out.shape == (R, eng.S)
    assert torch.equal(out[:, ts:ts + 4], (prefix + off).repeat_interleave(2, 0))
    assert ((out[:, ts + 4:] >= off) & (out[:, ts + 4:] < off + iv)).all()
    # the conditional rows carry the mapped captions, their unconditional twins the TL per-position pads
    assert torch.equal(smp.tokens[:R, :ts], smp._captions(text).repeat_interleave(2, 0))
    assert (smp.tokens[R:, :ts] == pads).all()
    g = smp.generate(text, temperature=0.0, guidance_scale=2.0)
    assert torch.equal(smp._uncond(B), pads.expand(B, ts))
    assert ((g[:, ts:] >= off) & (g[:, ts:] < off + iv)).all()
    assert torch.equal(smp.generate_graphed(text, temperature=0.0, guidance_scale=2.0), g)


# ================================================================================================== model_fn
EXTRA = {"image_position_embedding": "row_col", "per_position_padding": True, "padding_id": 299,
         "caption_dropout": 0.5}


def test_save_resume_and_cross_scheme_load(tmp_path):
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from test_loss_weights_gpu import _batch, _tiny_params
    img, cap = _batch()
    cap[:, 6:] = 299
    spec = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **EXTRA))
    eng = spec.engine
    assert eng.row_col and eng.per_position_padding and eng.V == 300 + 12 + 64 + 1
    toks = spec.assemble(img, cap)
    assert (toks[:, 6:12] == torch.arange(6, 12, device=DEV) + 300).all()
    for _ in range(2):
        spec.train_op(img, cap)
    state = spec.state_fn()
    assert "positional_embedding/image_row/adam_m" in state
    after = [spec.train_op(img, cap).clone() for _ in range(2)]
    resumed = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **EXTRA))
    resumed.load_fn(state)
    assert resumed.global_step == 2
    again = [resumed.train_op(img, cap).clone() for _ in range(2)]
    for a, b in zip(after, again):
        assert_same_bits(a.view(-1), b.view(-1), "loss after resume")
    assert_same_bits(resumed.engine.shadow, spec.engine.shadow, "bf16 parameters after resume")
    assert_same_bits(resumed.engine.pos_table.view(-1), spec.engine.pos_table.view(-1), "position table after resume")
    # a checkpoint of the other scheme names the variable that does not fit
    plain = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, padding_id=299, per_position_padding=True))
    with pytest.raises(L.DB200Error, match="positional_embedding/wpe"):
        plain.load_fn(state)
    with pytest.raises(L.DB200Error, match="positional_embedding/wpe"):
        spec.load_fn(plain.state_fn())
    no_pp = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, image_position_embedding="row_col"))
    with pytest.raises(L.DB200Error, match="embedding/wte"):
        no_pp.load_fn(state)


def test_zero1_on_one_gpu_equals_the_replicated_step_bitwise(ops):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    geom = (256, 2, 2, 300, 64, 24, 64)
    kw = dict(image_position_embedding="row_col", per_position_padding=True)
    for world in (2, 3):
        grp = Loopback(world)
        grp.engines = ranks = [DalleEngine(*geom, zero=grp.member(r), **kw) for r in range(world)]
        twin = DalleEngine(*geom, **kw)
        n = twin.n_params_padded
        twin.init_params(seed=5)
        for e in ranks:
            e.init_params(seed=5)
        # the replicated twin of tests/test_zero1_gpu.py: the full fp32 state P, M, V is stepped here, and the twin
        # runs on P with the vector parameters the ranks read (bf16-rounded), so both compute the same step
        P = twin.master[:n].clone()
        M, V = torch.zeros_like(P), torch.zeros_like(P)
        g = torch.Generator(device=DEV).manual_seed(world)
        for k in range(2):
            _twin_from(twin, P, ranks[0])
            for r, e in enumerate(ranks):
                assert_same_bits(e.shadow[:n], twin.shadow[:n], f"W={world} step {k}: rank {r} bf16 parameters")
                assert_same_bits(e.pos_table.view(-1), twin.pos_table.view(-1), f"W={world} step {k}: rank {r} table")
            tok = torch.randint(0, twin.V - 1, (world, twin.S), generator=g, device=DEV, dtype=I32)
            twin.zero_grads()
            for r, e in enumerate(ranks):
                e.zero_grads()
                e.forward(tok[r:r + 1], step=k, row0=r, global_batch=world)
                e.backward(1.0 / tok.numel())
                twin.forward(tok[r:r + 1], step=k, row0=r, global_batch=world)
                twin.backward(1.0 / tok.numel())
            grp.all_reduce_grads()
            G = ranks[0].grads[:n]
            assert_same_bits(G, twin.grads[:n], f"W={world} step {k}: reduced gradients")
            for e in ranks:
                e.optimizer_step(1e-3, clip=None)
            ops.adam_step(P, M, V, G, twin.shadow[:n], 1e-3, 0.9, 0.999, 1e-6, 0.0, None, 0.0, 1.0, False, 0)
            twin._compose_pos()
            for r, e in enumerate(ranks):
                assert_same_bits(e.shadow[:n], twin.shadow[:n], f"W={world} step {k}: rank {r} bf16 after the step")
                assert_same_bits(e.pos_table.view(-1), twin.pos_table.view(-1),
                                 f"W={world} step {k}: rank {r} table after the all-gather")
        exp = ranks[0].export_params()
        assert "positional_embedding/image_col" in exp and exp["positional_embedding/wpe"].shape == (24, 256)


@pytest.mark.parametrize("W", [2, 3])
def test_ranks_equal_one_rank_with_micro_batches_bitwise(rec, tmp_path, W):  # noqa: F811
    B = 12
    make = lambda **kw: _dalle_params(tmp_path, EXTRA, train_batch_size=B, **kw)      # noqa: E731
    p = make()
    feats, caps = _dalle_data(p, B, seed=W)
    caps[:, 7:] = 299
    ref, n, aux_off = _dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * _seq_len(p)), feats, caps, W)
    group, chk, (n_r, aux_r) = _dalle_ranks(rec, make, feats, caps, W, ref)
    assert (n_r, aux_r) == (n, aux_off)
    _check_coverage(group.trace, n, aux_off, len(ref))
    chk.assert_clean()


# ================================================================================================== command
def test_generate_dalle_end_to_end(tmp_path):
    import generate_dalle
    from PIL import Image
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.utils import save_checkpoint
    from dalle_mtf_b200.vae_engine import VaeEngine

    size, convblocks, K = 32, [[2, 64], [2, 128]], 64
    tv, ts, pad = 300, 12, 299
    vae_cfg = {"model_type": "vae", "dataset": {"image_size": size}, "num_tokens": K, "convblocks": convblocks,
               "model_path": str(tmp_path / "vae_run"), "use_bf16": True}
    dalle_cfg = {"model_type": "dalle", "dataset": {"image_size": size}, "predict_batch_size": 2,
                 "model_path": str(tmp_path / "dalle_run"), "n_embd": 256, "n_layers": 2, "n_heads": 2,
                 "text_vocab_size": tv, "image_vocab_size": K, "text_seq_len": ts,
                 "vae_model": str(tmp_path / "vae.json"), "padding_id": pad,
                 "image_position_embedding": "row_col", "per_position_padding": True}
    (tmp_path / "vae.json").write_text(json.dumps(vae_cfg))
    (tmp_path / "dalle.json").write_text(json.dumps(dalle_cfg))
    vae = VaeEngine(K, size, convblocks, 3, True, False, 1)
    vae.init_params(4)
    save_checkpoint(vae_cfg["model_path"], 7, {**{"vae/" + k: v for k, v in vae.export_params().items()},
                                               "global_step": 7})
    hw = size // 4
    eng = DalleEngine(256, 2, 2, tv, K, ts, hw * hw, image_position_embedding="row_col", per_position_padding=True)
    eng.init_params(5)
    save_checkpoint(dalle_cfg["model_path"], 3, {**eng.export_params(), "global_step": 3})
    caps = [[5, 6, 7], list(range(20, 32)), [pad, 1]]
    np.save(tmp_path / "caps.npy", np.array([c + [pad] * (ts - len(c)) for c in caps], dtype=np.int32))
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "dalle.json"), "--out", str(out), "--caption_ids",
                         str(tmp_path / "caps.npy"), "--samples_per_prompt", "2", "--guidance_scale", "2",
                         "--seed", "1"])
    pngs = sorted(p for p in os.listdir(out) if p.endswith(".png"))
    assert pngs == [f"{c:05d}_{s:02d}.png" for c in range(3) for s in range(2)]
    toks = np.load(out / "tokens.npy")
    off = tv + ts
    assert toks.shape == (6, ts + hw * hw)
    want = np.array([c + [pad] * (ts - len(c)) for c in caps])
    want = np.where(want == pad, tv + np.arange(ts)[None, :], want)
    assert (toks[:, :ts] == np.repeat(want, 2, 0)).all()
    assert ((toks[:, ts:] >= off) & (toks[:, ts:] < off + K)).all()
