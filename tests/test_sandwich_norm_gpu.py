"""Sandwich LayerNorm on the GPU: db200_layernorm_residual_fwd at every LayerNorm width and at the model shapes (its
statistics bit for bit db200_layernorm_fwd's, y within one bf16 ulp of float64), its argument checks, the GEMM's STORE
with dropout and no residual that now feeds it; the engine against oracle/dalle_sandwich.py (loss, loss rows, every
gradient, one Adam update), with each oracle mutant failing the same bounds; reproducibility, in-process ranks,
ZeRO-1; greedy, graphed, prefilled and guided decoding; checkpoints and their refusal across the key; the launches
with the key off, and a launch census of dalle_example plus the key whose new classes are replayed here."""
import math
import os

import pytest
import torch

from float64_bounds import DEV
from test_loss_weights_gpu import _engine, _step, _tiny_params, relfro

pytestmark = pytest.mark.gpu
BF16, F32, I32, F64 = torch.bfloat16, torch.float32, torch.int32, torch.float64
TAG = "sandwich_norm"
KEY = {"sandwich_norm": True}


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def _rand(rows, d, seed, scale=1.0, shift=0.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(rows, d, generator=g, device=DEV) * scale + shift).to(BF16)


def _vec(d, seed, base):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(d, generator=g, device=DEV) * 0.3 + base


def bf16_ulp(y):
    """The spacing of bf16 numbers at |y| (8 significant bits; subnormals ignored)."""
    e = torch.floor(torch.log2(y.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def check_residual_ln(ops, o, x, g, b, eps=1e-5, what=""):
    """layernorm_residual_fwd(o, x) against layernorm_fwd(o) (mean / rstd bit for bit) and against float64 from those
    statistics: |y - y64| <= one bf16 ulp of y64, plus the rounding of the fp32 evaluation's intermediates (a few fp32
    ulps of the largest terms x, (o - mean) rstd g and b, which can cancel)."""
    rows, d = o.shape
    y, mean, rstd = torch.empty_like(o), torch.empty(rows, dtype=F32, device=DEV), torch.empty(rows, dtype=F32,
                                                                                                device=DEV)
    ops.layernorm_residual_fwd(o, x, g, b, y, mean, rstd, eps)
    y0, mean0, rstd0 = torch.empty_like(o), torch.empty_like(mean), torch.empty_like(rstd)
    ops.layernorm_fwd(o, g, b, y0, mean0, rstd0, eps)
    torch.cuda.synchronize()
    assert torch.equal(mean, mean0) and torch.equal(rstd, rstd0), what
    n64 = (o.double() - mean.double()[:, None]) * rstd.double()[:, None] * g.double() + b.double()
    y64 = x.double() + n64
    terms = (o.double().abs() + mean.double().abs()[:, None]) * rstd.double()[:, None] * g.double().abs()
    slack = 4 * 2.0 ** -24 * (x.double().abs() + terms + b.double().abs())
    err = (y.double() - y64).abs()
    excess = (err - bf16_ulp(y64) - slack).max().item()
    assert excess <= 0, (what, excess)
    # the statistics themselves against float64
    o64 = o.double()
    m64 = o64.mean(1)
    r64 = torch.rsqrt(((o64 - m64[:, None]) ** 2).mean(1) + eps)
    assert relfro(mean, m64) < 1e-5 or (mean.double() - m64).abs().max().item() < 1e-5, what
    assert relfro(rstd, r64) < 1e-5, what
    return y


# ------------------------------------------------------------------------------------------------ kernel
WIDTHS = (256, 512, 768, 1024, 2048, 4096)
SHAPES = [(rows, d) for d in WIDTHS for rows in (8, 64, 37, 1000)] + \
    [(40960, 512), (10240, 1024), (5120, 4096)]       # dalle_example, dalle_coco and 12B token rows


@pytest.mark.parametrize("rows,d", SHAPES, ids=[f"{r}x{d}" for r, d in SHAPES])
def test_residual_layernorm_matches_layernorm_stats_and_float64(ops, rows, d):
    from dalle_mtf_b200.dalle_engine import LAYERNORM_WIDTHS
    assert set(WIDTHS) == set(LAYERNORM_WIDTHS)
    o = _rand(rows, d, rows + d, scale=3.0, shift=0.5)
    x = _rand(rows, d, rows + d + 1, scale=2.0)
    check_residual_ln(ops, o, x, _vec(d, d, 1.0), _vec(d, d + 1, 0.0), what=f"{rows}x{d}")
    print(f"[{TAG}] layernorm_residual_fwd {rows} x {d}: stats bit for bit, y within 1 bf16 ulp of float64")


def test_residual_layernorm_edge_values(ops):
    """Constant rows (variance 0: rstd = 1/sqrt(eps)), large offsets, a residual that cancels the normalised row, and
    y written in place over the residual."""
    d, rows = 512, 64
    o = _rand(rows, d, 1, scale=2.0)
    o[:8] = 3.0
    o[8:16] = (o[8:16].float() * 0.01 + 100.0).to(BF16)
    x = _rand(rows, d, 2)
    g, b = _vec(d, 3, 1.0), _vec(d, 4, 0.0)
    y = check_residual_ln(ops, o, x, g, b, what="edge")
    yi = x.clone()
    mean, rstd = torch.empty(rows, dtype=F32, device=DEV), torch.empty(rows, dtype=F32, device=DEV)
    ops.layernorm_residual_fwd(o, yi, g, b, yi, mean, rstd)
    torch.cuda.synchronize()
    assert torch.equal(yi.view(torch.int16), y.view(torch.int16))


def test_entry_point_refuses_bad_arguments(ops):
    from dalle_mtf_b200 import lib as L
    lib = L.load()
    rows, d = 8, 256
    o, x, y = _rand(rows, d, 0), _rand(rows, d, 1), torch.zeros(rows, d, dtype=BF16, device=DEV)
    g, b = torch.ones(d, device=DEV), torch.zeros(d, device=DEV)
    mean, rstd = torch.zeros(rows, device=DEV), torch.zeros(rows, device=DEV)
    s = L.stream_ptr()
    P = [o.data_ptr(), x.data_ptr(), g.data_ptr(), b.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr()]
    E_INV, E_ALIGN, E_UNSUP = -1, -2, -4
    for k in range(7):
        args = list(P)
        args[k] = None
        assert lib.db200_layernorm_residual_fwd(s, *args, rows, d, 1e-5) == E_INV, k
    for k in range(5):
        args = list(P)
        args[k] += 2
        assert lib.db200_layernorm_residual_fwd(s, *args, rows, d, 1e-5) == E_ALIGN, k
    assert lib.db200_layernorm_residual_fwd(s, *P, 0, d, 1e-5) == E_INV
    for bad_d in (128, 300, 8192):
        assert lib.db200_layernorm_residual_fwd(s, *P, rows, bad_d, 1e-5) == E_UNSUP
    torch.cuda.synchronize()
    assert not y.any() and not mean.any() and not rstd.any()                     # nothing ran
    for call in (lambda: ops.layernorm_residual_fwd(o, x[:4], g, b, y, mean, rstd),
                 lambda: ops.layernorm_residual_fwd(o, x, g[:128], b, y, mean, rstd),
                 lambda: ops.layernorm_residual_fwd(o.float(), x, g, b, y, mean, rstd),
                 lambda: ops.layernorm_residual_fwd(o, x, g, b, y, mean[:4], rstd)):
        with pytest.raises(L.DB200Error):
            call()


@pytest.mark.parametrize("M,N,K", [(40960, 512, 512), (40960, 512, 2048), (10240, 1024, 4096), (5120, 4096, 4096),
                                   (5120, 4096, 16384), (200, 256, 1024)])
def test_gemm_store_with_dropout_takes_a_null_residual(ops, M, N, K):
    """The Wo / W2 products of a sandwich layer store drop(x w + bias) without a residual: equal to the same product
    with a zero residual, and within float64 bounds of keep * scale * (x w + bias)."""
    from dalle_mtf_b200 import lib as L
    x, w = _rand(M, K, M + K, scale=0.5), _rand(K, N, K + N, scale=0.05)
    bias = _vec(N, N, 0.0)
    site = L.make_dropout(0.2, 5, 3, L.dropout_site_mlp_out(1), 7)
    out, ref = torch.empty(M, N, dtype=BF16, device=DEV), torch.empty(M, N, dtype=BF16, device=DEV)
    ops.linear_fwd(x, w, out, bias=bias, dropout=site)
    ops.linear_fwd(x, w, ref, bias=bias, residual=torch.zeros(M, N, dtype=BF16, device=DEV), dropout=site)
    keep = torch.empty(M, N, dtype=torch.uint8, device=DEV)
    ops.dropout_mask(site, L.DROPOUT_ELEMENTWISE, (M, N), keep)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    want = (x.double() @ w.double() + bias.double()) * keep.double() / 0.8
    e = relfro(out, want)
    assert e < 1e-2, e
    assert not out[keep == 0].any()


# ------------------------------------------------------------------------------------------------ engine vs oracle
MIXED = ["axial_row", "axial_col", "conv", "local"]


def _sandwich_vs_oracle(types=None, B=3, seed=1, d=256, H=2, ts=24, W=8, recompute=False, rates=None, row_col=False,
                        mask=False, act="relu", gated=False, rotary=None, shift=False, weights=None, adam=False,
                        mutants=(), tv=300, iv=64):
    """One sandwich engine step (forward, backward) against oracle/dalle_sandwich.py in fp32 (the bounds) and with
    the reference's bf16 policy (the gradient scale): loss within 1e-3, loss rows within 5e-3, every gradient (the 4 L
    norm vectors included) within 1.25 x the bf16 oracle's error + 1e-2 (tests/test_shift_tokens_gpu.py's bounds);
    adam: one optimiser step against oracle/optim.py.  Each mutant's fp32 oracle must violate one of the bounds."""
    import conv_oracle as OC
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle_glu as OGL
    from oracle import dalle_input as I
    from oracle import dalle_sandwich as OSW
    from oracle import logits_mask as OLM
    from test_parity_baseline_gpu import _randomise_small_params
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    isl = W * W
    types = list(types or ["global", "global"])
    nl = len(types)
    cfg = OC.ConvConfig(d, nl, H, tv, iv, ts, isl, attention_types=tuple(types), local_attention_radius=8,
                        conv_attention_kernel=3)
    inp = I.InputConfig("row_col" if row_col else "absolute", False, None)
    params = I.init_params(cfg, inp, seed)
    g = torch.Generator().manual_seed(seed + 1)
    _randomise_small_params(params, g)
    if gated:
        params = OGL.init_params(params, cfg, seed + 7)
    params = OSW.init_params(params, cfg, seed + 11)            # random g / b: swapped norms must show
    text = torch.randint(0, tv - 1, (B, ts), generator=g)
    tokens = I.assemble(text, torch.randint(0, iv, (B, isl), generator=g), cfg, inp)
    step = 3 if rates else None
    dropout = ((rates,) * 3, seed, step, 0) if rates else None
    off, _ = I.vocab(cfg, inp)
    w, z = weights if weights else (None, 0.0)

    def oracle(bf16, mutate=None):
        base = lambda p, t, c, dr, bf16=False, quirks=None: OSW.forward(  # noqa: E731
            p, t, c, dr, bf16=bf16, quirks=quirks, layers=OC, activation=act, gated=gated, rotary=rotary,
            shift_tokens=shift, sandwich_mutate=mutate)
        if not mask and weights is None:
            loss, rows, _, grads = I.loss_and_grads(params, tokens, cfg, inp, dropout, bf16, base=base)
            return loss, rows, grads
        fwd = lambda p, t: I.forward(p, t, cfg, inp, dropout, bf16, base=base)  # noqa: E731
        loss, rows, _, _, grads = OLM.loss_and_grads(params, tokens, I._model_cfg(cfg, inp), off, weights=w, z=z,
                                                     forward=fwd, mask=mask)
        return loss, rows, grads

    loss32, rows32, g32 = oracle(False)
    _, _, g16 = oracle(True)
    kw = dict(rotary_dim=rotary[0], rotary_base=rotary[1]) if rotary else {}
    if weights:
        kw.update(loss_weights=w, z_loss=z)
    eng = DalleEngine(d, nl, H, tv, iv, ts, isl, recompute_grad=recompute, attention_types=types,
                      local_attention_radius=8, conv_attention_kernel=3, dropout=(rates or 0.0,) * 3,
                      dropout_seed=seed, image_position_embedding=inp.image_position_embedding, activation=act,
                      gated_mlp=gated, logits_mask=mask, shift_tokens=shift, sandwich_norm=True, **kw)
    eng.load_params(params)
    tok = tokens.to(I32).to(DEV)
    T = tok.numel()
    eng.zero_grads()
    acc = eng.forward(tok, step=step)
    if weights:
        eng.backward(1.0)
        torch.cuda.synchronize()
        loss = acc[0].item()
    else:
        eng.backward(1.0 / T)
        torch.cuda.synchronize()
        loss = acc.item() / T
    rows = eng._bufs["loss_rows"].view(B, -1).clone()
    grads = eng.export_params(eng.grads)
    assert set(OSW.norm_names(nl)) <= set(grads)

    def violations(l32, r32, gg32):
        bad, worst = [], [0.0, None]

        def bound(name, err, limit):
            if err > limit:
                bad.append((name, err, limit))
            if err / limit > worst[0]:
                worst[:] = [err / limit, name]
        bound("loss", abs(loss - l32.item()), 1e-3 * abs(l32.item()))
        bound("loss_rows", relfro(rows, r32), 5e-3)
        for k in gg32:
            if g32[k].any():
                bound("grad " + k, relfro(grads[k], gg32[k]), 1.25 * relfro(g16[k], g32[k]) + 1e-2)
        return bad, worst

    bad, worst = violations(loss32, rows32, g32)
    print(f"[{TAG}] engine d {d} types {types} recompute {recompute} rates {rates} row_col {row_col} mask {mask} {act} "
          f"gated {gated} rotary {rotary} shift {shift} weights {weights}: loss {loss:.6f} oracle {loss32.item():.6f}, "
          f"worst err/bound {worst[0]:.4f} ({worst[1]}), violations {bad}")
    assert not bad
    for m in mutants:
        ml, mr, mg = oracle(False, m)
        mbad, _ = violations(ml, mr, mg)
        print(f"[{TAG}]   mutant {m}: {len(mbad)} violated bounds, e.g. {mbad[:2]}")
        assert mbad, m
    if adam:
        from oracle import optim as OO
        hp = {"lr": 1e-3, "train_steps": 1000, "warmup_steps": 10}
        zeros = {k: torch.zeros_like(v) for k, v in params.items()}
        newp, _, _, lr, gn = OO.dalle_train_step(params, zeros, zeros, grads, 5, hp)
        eng.optimizer_step(lr)
        torch.cuda.synchronize()
        assert abs(eng.gnorm_sq.sqrt().item() - gn.item()) <= 1e-4 * gn.item()
        after = eng.export_params()
        for k in params:
            if (newp[k] - params[k]).norm() > 0:
                assert relfro(after[k] - params[k], newp[k] - params[k]) <= 1e-3, k


def test_engine_matches_the_oracle_and_not_its_mutants():
    _sandwich_vs_oracle(adam=True, mutants=("post_ln", "swapped", "ignored"))


def test_dalle_example_geometry_matches_the_oracle():
    """The dalle_example layer (d 512, 4 heads, TL 256, a 32 x 32 grid, the GPT-2 text vocabulary), one sequence."""
    _sandwich_vs_oracle(["global", "global"], B=1, seed=5, d=512, H=4, ts=256, W=32, tv=50258, iv=512,
                        mutants=("swapped", "ignored"))


def test_a_12b_width_layer_with_recompute_matches_the_oracle():
    _sandwich_vs_oracle(["global"], B=2, seed=6, d=4096, H=32, ts=8, W=4, recompute=True, mutants=("ignored",))


@pytest.mark.parametrize("variant", [dict(rates=0.1), dict(rates=0.1, recompute=True),
                                     dict(gated=True, act="gelu", rotary=(64, 10000.0), shift=True),
                                     dict(mask=True), dict(weights=((1.0, 7.0), 1e-4)), dict(types=MIXED),
                                     dict(row_col=True)],
                         ids=["dropout", "dropout_recompute", "geglu_rotary_shift", "logits_mask", "weighted",
                              "mixed", "row_col"])
def test_engine_variants_match_the_oracle_and_not_its_mutants(variant):
    mutants = ("norm_before_drop", "swapped") if variant.get("rates") else ("swapped", "post_ln")
    _sandwich_vs_oracle(seed=3 if variant.get("types") else 2, mutants=mutants, **variant)


# ------------------------------------------------------------------------------------------------ steps
def _small(seed=0, sandwich=True):
    from oracle import dalle as O
    from oracle import dalle_sandwich as OSW
    cfg = O.DalleConfig(256, 2, 2, 300, 60, 40, 64)
    params = O.init_params(cfg, seed)
    if sandwich:
        params = OSW.init_params(params, cfg, seed + 5)
    g = torch.Generator().manual_seed(seed + 1)
    tokens = torch.cat([torch.randint(0, 300, (4, 40), generator=g), torch.randint(300, 360, (4, 64), generator=g)], 1)
    return cfg, params, tokens.to(I32).to(DEV)


def test_sandwich_steps_are_bit_identical_and_micro_batches_match():
    cfg, params, tok = _small(3)
    eng = _engine(cfg, sandwich_norm=True, attention_types=["global", "axial_col"], dropout=(0.1, 0.1, 0.1))
    eng.load_params(params)

    def step(split=1):
        eng.zero_grads()
        mb = tok.shape[0] // split
        for i in range(split):
            eng.forward(tok[i * mb:(i + 1) * mb], step=4, row0=i * mb)
            eng.backward(1.0 / tok.numel())
        torch.cuda.synchronize()
        return eng.grads.clone()
    a, b = step(), step()
    assert torch.equal(a, b)
    n = eng.n_params_padded
    assert relfro(step(2)[:n], a[:n]) < 1e-5


def test_in_process_ranks_equal_one_rank_with_micro_batches_bitwise(monkeypatch, tmp_path):
    """tests/test_data_parallel_gpu.py's criterion for the plain step (bit for bit), with the key and every feature."""
    from test_data_parallel_gpu import FEATURES, _Rec, _check_coverage, _dalle_data, _dalle_params, _dalle_ranks, \
        _dalle_reference, _seq_len, STEPS
    rec = _Rec(monkeypatch)
    extra = dict(FEATURES, **KEY)
    W, B = 2, 12
    make = lambda **kw: _dalle_params(tmp_path, extra, train_batch_size=B, **kw)      # noqa: E731
    p = make()
    feats, caps = _dalle_data(p, B, seed=W)
    ref, n, aux_off = _dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * _seq_len(p)), feats, caps, W)
    group, chk, (n_r, aux_r) = _dalle_ranks(rec, make, feats, caps, W, ref)
    assert (n_r, aux_r) == (n, aux_off)
    _check_coverage(group.trace, n, aux_off, STEPS)
    chk.assert_clean()


@pytest.mark.parametrize("world", [2, 3])
def test_zero1_sandwich_step_equals_the_replicated_step_bitwise(world):
    from test_zero1_gpu import Loopback, _twin_from, assert_same_bits
    cfg, params, tok = _small(11)
    # bf16-representable values: the replicated twin starts its vector parameters from the ZeRO engine's bf16 copy,
    # so its Adam step agrees bit for bit only when the fp32 masters agree too
    params = {k: v.to(BF16).float() for k, v in params.items()}
    grp = Loopback(world)
    grp.engines = ranks = [_engine(cfg, zero=grp.member(r), **KEY) for r in range(world)]
    twin = _engine(cfg, **KEY)
    for e in [twin] + ranks:
        e.load_params(params)
    n = twin.n_params_padded
    _twin_from(twin, twin.master[:n].clone(), ranks[0])
    g_ref = _step(twin, tok)
    for r, e in enumerate(ranks):
        assert_same_bits(_step(e, tok), g_ref, f"ZeRO-1 rank {r} sandwich gradients")
    twin.optimizer_step(1e-3)
    for e in ranks:
        e.optimizer_step(1e-3)
    for r, e in enumerate(ranks):
        assert_same_bits(e.shadow[:n], twin.shadow[:n], f"ZeRO-1 rank {r} parameters after the step")
    ex = ranks[0].export_params()
    for k, v in twin.export_params().items():
        assert torch.equal(ex[k], v.to(BF16).float()), k


# ------------------------------------------------------------------------------------------------ generation
def _sharp_sandwich_engine(d, Lyr, H, tv, iv, ts, isl, **kw):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    from oracle import dalle_sandwich as OSW
    cfg = O.DalleConfig(d, Lyr, H, tv, iv, ts, isl)
    params = OSW.init_params(O.init_params(cfg, 3), cfg, 4)
    g = torch.Generator().manual_seed(9)
    for k in params:
        if k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if "wte" in k or "wout" in k or k.endswith("kernel"):
            params[k] = params[k] * 4
    eng = DalleEngine(d, Lyr, H, tv, iv, ts, isl, sandwich_norm=True, **kw)
    eng.load_params(params)
    return eng


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_decoding_follows_the_full_forward_and_the_prefill():
    from dalle_mtf_b200.sampling import DalleSampler
    from test_prefill_gpu import greedy_agrees_with_full_forward
    ts, W = 16, 8
    S = ts + W * W
    eng = _sharp_sandwich_engine(256, 4, 2, 300, 64, ts, W * W, attention_types=["global", "axial_col", "conv",
                                                                                  "axial_row"])
    g = torch.Generator().manual_seed(4)
    text = torch.randint(0, 299, (3, ts), generator=g).to(I32).to(DEV)
    smp = DalleSampler(eng)
    out, step_logits = smp.generate(text, 0.0, return_logits=True)
    assert torch.equal(smp.generate_graphed(text, temperature=0.0), out)
    greedy_agrees_with_full_forward(eng, out, ts)
    full = eng.logits(out)
    e = relfro(torch.stack(step_logits, 1), full[:, :S - 1])
    assert e < 2e-2, e
    smp.generate(text, 0.0)
    eager_k = [c.clone() for c in smp.kc]
    for P in (ts, ts + W + 3, S - 1):
        kc = [torch.zeros_like(c) for c in smp.kc]
        vc = [torch.zeros_like(c) for c in smp.vc]
        logits = eng.prefill(out[:, :P].contiguous(), kc, vc).clone()
        assert _bits_equal(kc[0][:, :P], eager_k[0][:, :P]), P                    # layer 0's keys: bit for bit
        for i in range(1, len(kc)):
            ei = relfro(kc[i][:, :P], eager_k[i][:, :P])
            assert ei < 2e-2, (P, i, ei)
        ep = relfro(logits[:, :eng.V], step_logits[P - 1])
        print(f"[{TAG}] decode vs full {e:.2e}, prefill P={P} vs decoding {ep:.2e}")
        assert ep < 2e-2, ep
    done = smp.complete(text, out[:, ts:ts + W + 3].contiguous() - eng.image_offset, temperature=0)
    greedy_agrees_with_full_forward(eng, done, ts + W + 3)
    torch.manual_seed(0)
    guided = smp.complete(text[:2], out[:2, ts:ts + W + 3].contiguous() - eng.image_offset, samples_per_prompt=2,
                          guidance_scale=3.0, top_k=16)
    assert guided.shape == (4, S)
    assert ((guided[:, ts:] >= eng.image_offset) & (guided[:, ts:] < eng.image_offset + 64)).all()
    gg = smp.generate_graphed(text[:2], temperature=0.0, guidance_scale=2.0)
    ge = smp.generate(text[:2], 0.0, guidance_scale=2.0)
    assert torch.equal(gg, ge)


# ------------------------------------------------------------------------------------------------ checkpoints
def test_export_load_round_trip_and_mismatched_checkpoints_are_refused():
    from dalle_mtf_b200 import lib as L
    from oracle import dalle_sandwich as OSW
    cfg, params, tok = _small(7)
    eng = _engine(cfg, **KEY)
    eng.load_params(params)
    ex = eng.export_params()
    assert set(ex) == set(params)
    for k in params:
        assert torch.equal(ex[k], params[k].float()), k
    plain_params = {k: v for k, v in params.items() if "/norm_out/" not in k}
    with pytest.raises(L.DB200Error, match="layer_0/attn/norm_out/g"):
        eng.load_params(plain_params)
    plain = _engine(cfg)
    with pytest.raises(L.DB200Error, match="layer_0/attn/norm_out/g"):
        plain.load_params(params)
    with pytest.raises(L.DB200Error, match="layer_1/mlp/norm_out/b"):
        eng.load_params({k: v for k, v in params.items() if k != "layer_1/mlp/norm_out/b"})
    plain.load_params(plain_params)
    assert set(plain.export_params()) == set(plain_params)
    assert set(OSW.norm_names(cfg.n_layers)) == set(params) - set(plain_params)


def _batch():
    g = torch.Generator().manual_seed(3)
    return torch.rand(4, 16, 16, 3, generator=g) * 2 - 1, torch.randint(0, 299, (4, 12), generator=g)


def test_model_fn_checkpoint_resumes_bit_exactly_and_dalle_takes_the_key(tmp_path):
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.models import DALLE
    img, cap = _batch()
    plain = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path))
    sw = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **KEY))
    assert sw.engine.sandwich_norm and not plain.engine.sandwich_norm
    assert sw.engine.n_params() - plain.engine.n_params() == 4 * 256 * 2
    sw.train_op(img, cap)
    st = sw.state_fn()
    assert {k for k in st if "/norm_out/" in k and not k.endswith(("adam_m", "adam_v"))} == \
        {f"layer_{i}/{b}/norm_out/{v}" for i in range(2) for b in ("attn", "mlp") for v in "gb"}
    a = sw.train_op(img, cap).clone()
    sa = [t.clone() for t in (sw.engine.master, sw.engine.adam_m, sw.engine.adam_v)]
    resumed = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **KEY))
    resumed.load_fn(st)
    b = resumed.train_op(img, cap)
    assert torch.equal(a, b)
    for x, y in zip(sa, (resumed.engine.master, resumed.engine.adam_m, resumed.engine.adam_v)):
        assert torch.equal(x, y)
    with pytest.raises(L.DB200Error, match="norm_out"):
        plain.load_fn(st)
    m = DALLE(256, text_vocab_size=300, image_vocab_size=60, text_seq_len=40, image_seq_len=64, n_layers=1, n_heads=2,
              mode="eval", params=KEY)
    assert m.engine.sandwich_norm
    g = torch.Generator().manual_seed(9)
    tokens = torch.cat([torch.randint(0, 300, (2, 40), generator=g), torch.randint(300, 360, (2, 64), generator=g)], 1)
    loss, loss_batch = m.forward({"tokens": tokens})
    assert math.isfinite(loss.item()) and loss_batch.shape == (2, 104)


def test_generate_cli_runs_on_a_tiny_sandwich_model(tmp_path):
    import json
    import numpy as np
    import generate_dalle
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.utils import save_checkpoint
    img, cap = _batch()
    p = _tiny_params(tmp_path, **KEY)
    spec = dalle_model_fn(img, cap, "train", p)
    spec.train_op(img, cap)
    vae = spec.extra["vae"]
    save_checkpoint(str(tmp_path / "vae"), 1, {"vae/" + k: v for k, v in vae.export_params().items()})
    save_checkpoint(str(tmp_path / "dalle"), 1, spec.state_fn())
    vcfg = dict(p["vae_params"], model_path=str(tmp_path / "vae"))
    (tmp_path / "vae.json").write_text(json.dumps(vcfg))
    cfg = {k: v for k, v in p.items() if k != "vae_params"}
    cfg.update(vae_model=str(tmp_path / "vae.json"), model_path=str(tmp_path / "dalle"), predict_batch_size=2)
    (tmp_path / "sw.json").write_text(json.dumps(cfg))
    np.save(tmp_path / "ids.npy", np.array([[1, 2, 3] + [299] * 9, [4, 5] + [299] * 10], dtype=np.int64))
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "sw.json"), "--caption_ids", str(tmp_path / "ids.npy"),
                         "--out", str(out), "--temperature", "0"])
    toks = np.load(out / "tokens.npy")
    assert toks.shape == (2, spec.engine.S) and len(list(out.glob("*.png"))) == 2


# ------------------------------------------------------------------------------------------------ launches
@pytest.mark.parametrize("recompute", [False, True], ids=["saved", "recompute"])
def test_key_off_launches_what_it_launched_before(monkeypatch, recompute):
    """With the key absent or false, forward, backward and the optimiser step call the same ops in the same order
    with the same launch count; with it on, 2 L layernorm_residual_fwd (4 L with recompute_grad) and 2 L more
    layernorm_bwd calls are added."""
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops as O
    cfg, params, tok = _small(10, sandwich=False)
    _, sparams, _ = _small(10)
    calls = []
    names = [n for n, f in vars(O).items() if callable(f) and not n.startswith("_") and getattr(f, "__module__", "")
             == O.__name__]
    for n in names:
        f = getattr(O, n)
        monkeypatch.setattr(O, n, (lambda n, f: lambda *a, **k: (calls.append(n), f(*a, **k))[1])(n, f))
    seqs, counts = [], []
    for kw in ({}, {"sandwich_norm": False}, KEY):
        eng = _engine(cfg, recompute_grad=recompute, **kw)
        eng.load_params(sparams if kw.get("sandwich_norm") else params)
        _step(eng, tok, 1.0 / tok.numel())
        calls.clear()
        n0 = L.launch_count()
        _step(eng, tok, 1.0 / tok.numel())
        eng.optimizer_step(1e-3)
        torch.cuda.synchronize()
        counts.append(L.launch_count() - n0)
        seqs.append(list(calls))
    Lyr = cfg.n_layers
    assert seqs[0] == seqs[1] and counts[0] == counts[1]
    assert "layernorm_residual_fwd" not in seqs[0]
    n_fwd = seqs[2].count("layernorm_residual_fwd")
    assert n_fwd == (4 if recompute else 2) * Lyr
    assert seqs[2].count("layernorm_bwd") == seqs[0].count("layernorm_bwd") + 2 * Lyr


def _ln_bwd_reference(dy, x, g, mean, rstd, dres):
    """float64 LayerNorm backward from the kernel's statistics: dx = rstd (dy g - mean(dy g) - xhat mean(dy g xhat))
    [+ dres], dg = sum dy xhat, db = sum dy."""
    xh = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    t = dy.double() * g.double()
    dx = (t - t.mean(1, keepdim=True) - xh * (t * xh).mean(1, keepdim=True)) * rstd.double()[:, None]
    if dres is not None:
        dx = dx + dres.double()
    return dx, (dy.double() * xh).sum(0), dy.double().sum(0)


def _replay_optimizer_class(ops, entry, f):
    from test_zero1_gpu import LR, _adam_f64_slabs
    n = f["n"] if entry != "cast_f32_to_bf16" else f["src"][0][0]
    gen = torch.Generator(device=DEV).manual_seed(n)
    rnd = lambda s=1.0: torch.randn(n, generator=gen, device=DEV) * s  # noqa: E731
    if entry == "cast_f32_to_bf16":
        src, dst = rnd(), torch.empty(n, dtype=BF16, device=DEV)
        ops.cast_f32_to_bf16(src, dst)
        torch.cuda.synchronize()
        assert torch.equal(dst, src.to(BF16))
        return
    g = rnd(1e-3)
    gn = torch.zeros(1, device=DEV)
    ops.sqnorm(g, gn)
    torch.cuda.synchronize()
    assert abs(gn.item() - (g.double() ** 2).sum().item()) <= 1e-5 * gn.item()
    if entry == "sqnorm":
        return
    assert not f["wd"] and not f["bias_correction"], f
    p, m, v = rnd(0.02), rnd(1e-4), rnd(1e-4).abs() * 1e-4
    before = (p.clone(), m.clone(), v.clone(), g.clone())
    p16 = torch.empty(n, dtype=BF16, device=DEV)
    clip = 1.0 if f["clip"] else 0.0
    ops.adam_step(p, m, v, g, p16, LR, 0.9, 0.999, 1e-6, 0.0, gn if f["clip"] else None, clip, 1.0, False, 0,
                  zero_grad=f["zero_grad"])
    torch.cuda.synchronize()
    _adam_f64_slabs(f"adam_step n={n}", before, (p, m, v, p16), gn.item(), clip)
    if f["zero_grad"]:
        assert not g.any()


def test_launch_census_of_a_sandwich_model_replays_its_new_classes(ops, monkeypatch):
    """dalle_example_b200 with and without the key recorded by test_dalle_config_launches_gpu.py's recorder (train,
    eval, eager and graphed decoding, prefill with guidance): the sandwich model launches the plain model's classes
    plus layernorm_residual_fwd, layernorm_bwd and gemm classes, and the optimiser's sqnorm / adam_step /
    cast_f32_to_bf16 at the parameter count the 4 L new vectors change, each replayed here at its recorded shape
    against float64 (the cast bit for bit against torch)."""
    import launch_census as LC
    import test_dalle_config_launches_gpu as CL
    import test_dalle_kernels_gpu as DK
    from dalle_mtf_b200 import lib as L
    base = DK._config("dalle_example_b200")
    recorded = {}
    for name, extra in (("plain", {}), ("sandwich", KEY)):
        monkeypatch.setattr(DK, "_config", lambda c, extra=extra: dict(base, **extra))
        recorded[name] = set(CL.record_config("dalle_example_b200")[0])
    added = recorded["sandwich"] - recorded["plain"]
    entries = {c[0] for c in added}
    assert "layernorm_residual_fwd" in entries and entries <= {"layernorm_residual_fwd", "layernorm_bwd", "gemm",
                                                               "sqnorm", "adam_step", "cast_f32_to_bf16"}, entries
    for c in sorted(added, key=repr):
        f = LC.fields(c)
        if c[0] == "layernorm_residual_fwd":
            (rows, d), _ = f["o"]
            o, x = _rand(rows, d, rows, scale=2.0), _rand(rows, d, rows + 1)
            check_residual_ln(ops, o, x, _vec(d, 1, 1.0), _vec(d, 2, 0.0), what=repr(c))
        elif c[0] in ("sqnorm", "adam_step", "cast_f32_to_bf16"):
            _replay_optimizer_class(ops, c[0], f)
        elif c[0] == "layernorm_bwd":
            rows, d = f["rows"], f["d"]
            x, dy = _rand(rows, d, rows, scale=2.0), _rand(rows, d, rows + 1)
            dres = _rand(rows, d, rows + 2) if f["dres"] else None
            g = _vec(d, 3, 1.0)
            mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
            ops.layernorm_fwd(x, g, torch.zeros(d, device=DEV), torch.empty_like(x), mean, rstd)
            dx, dg, db = torch.empty_like(x), torch.zeros(d, device=DEV), torch.zeros(d, device=DEV)
            dxsum = torch.zeros(d, device=DEV) if f["dxsum"] else None
            site = L.make_dropout(0.1, 1, 2, L.dropout_site_mlp_out(0), 0) if f["dropout"] else None
            dxm = torch.empty_like(x) if site is not None else None
            ops.layernorm_bwd(dy, x, g, mean, rstd, dres, dx, dg, db, dxsum=dxsum, dxm=dxm, dropout=site)
            torch.cuda.synchronize()
            rdx, rdg, rdb = _ln_bwd_reference(dy, x, g, mean, rstd, dres)
            assert relfro(dx, rdx) < 1e-2 and relfro(dg, rdg) < 1e-4 and relfro(db, rdb) < 1e-4, c
            if dxsum is not None:
                assert relfro(dxsum, (dxm if dxm is not None else dx).double().sum(0)) < 1e-4, c
        else:
            M, N, K = f["M"], f["N"], f["K"]
            assert not f["residual"] and f["mode"] == L.EPI_STORE and not f["a_mn"] and f["b_mn"], c
            x, w = _rand(M, K, M, scale=0.5), _rand(K, N, K, scale=0.05)
            bias = _vec(N, N, 0.0) if f["bias"] else None
            site = L.make_dropout(0.1, 1, 2, L.dropout_site_attn_out(0), 0) if f["dropout"] else None
            out = torch.empty(M, N, dtype=BF16, device=DEV)
            ops.linear_fwd(x, w, out, bias=bias, dropout=site)
            want = x.double() @ w.double() + (bias.double() if bias is not None else 0)
            if site is not None:
                keep = torch.empty(M, N, dtype=torch.uint8, device=DEV)
                ops.dropout_mask(site, L.DROPOUT_ELEMENTWISE, (M, N), keep)
                want = want * keep.double() / 0.9
            torch.cuda.synchronize()
            assert relfro(out, want) < 1e-2, c
        print(f"[{TAG}] census class {c[0]} {f}: replayed against float64")
