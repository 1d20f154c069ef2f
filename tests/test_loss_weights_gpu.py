"""GPU tests of the weighted cross-entropy (text_loss_weight / image_loss_weight / z_loss).

Kernels: CE_STATS -> db200_ce_finish_weighted -> db200_gemm_bf16_ce_weighted against float64 on the same bf16 operands,
per element, with the bounds of test_dalle_kernels_gpu.py's cross-entropy (its module docstring) extended by the row
coefficient c = a (1 + 2 z lse):
  loss_rows = CE + z lse^2 adds z (2 |lse| eps_lse + 3 U lse^2);
  dlogits_j = a ((1 + 2 z lse) p_j - [j = label]):  |err| <= 1.01 |c| p_j (delta_j + eps_lse + eps_exp_j)
      + 2 a z eps_lse p_j + 4 U |c| p_j + U a [j = label] + half a bf16 ulp,  eps_exp_j with 2 U |ln |c|| in place of
      2 U |ln alpha|;
  the four sums add the row bounds plus (T/32 + 48) U of the sums of absolute values.
A zero-weight class must get exact zeros; a mutant oracle (class boundary at TL, or the z gradient without its factor
2) must fail the same bounds.

Engine: the weighted step against oracle/loss_weights.py, against the unweighted step, bit-reproducibility,
micro-batching, reserved SMs, 2 ranks, eval_op and DALLE.forward.
"""
import math
import os

import pytest
import torch

import float64_bounds
from float64_bounds import DEV, U, UTC, nan_like
from test_dalle_kernels_gpu import Worst, _config, _gen, _slabs, ce_operands, check, synthetic_tokens

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def run_weighted_ce(ops, tag, T, K, V, Vpad, S, TL, *, labels, h, W, bias, weights, z, global_batch=None,
                    mutants=(), dl=None):
    """CE_STATS -> ce_finish_weighted -> weighted CE_GRAD, checked per element in row slabs; returns the worst
    err/bound.  mutants: oracle.loss_weights LossQuirks whose dlogits must exceed the bound somewhere.  dl: the
    NaN-filled [T, Vpad] bf16 gradient to write (default: a fresh one)."""
    from dalle_mtf_b200 import lib as L
    from oracle import loss_weights as OW
    IL = S - TL
    Bg = T // S if global_batch is None else global_batch
    a_text, a_image = OW.coefficients(weights, TL, IL, Bg)
    cew = L.make_ce_weights(S, TL - 1, a_text, a_image, z)
    nt = ops.ce_tiles(Vpad)
    pm, ps = nan_like((nt, T), F32), nan_like((nt, T), F32)
    ll, lse, lr = nan_like((T,), F32), nan_like((T,), F32), nan_like((T,), F32)
    base = torch.tensor([0.5, 0.25, -0.75, 0.125], device=DEV)
    sums = base.clone()
    ops.gemm(h, W, None, T, Vpad, K, a_mn=False, b_mn=True, mode=L.EPI_CE_STATS, bias=bias, labels=labels,
             part_max=pm, part_sum=ps, label_logit=ll, n_valid=V)
    ops.ce_finish_weighted(pm, ps, ll, lse, lr, sums, cew)
    del pm, ps
    dl = nan_like((T, Vpad), BF16) if dl is None else dl
    cs_base = torch.randn(Vpad, generator=_gen(T + Vpad), device=DEV) * 1e-3
    cs = cs_base.clone()
    ops.gemm(h, W, dl, T, Vpad, K, a_mn=False, b_mn=True, mode=L.EPI_CE_GRAD, bias=bias, labels=labels, lse=lse,
             n_valid=V, colsum=cs, ce_weights=cew)
    W64, b64 = W[:, :V].to(F64), bias[:V].to(F64)
    Wa = W64.abs()
    a32 = torch.tensor([cew.a_text, cew.a_image], dtype=F64, device=DEV)   # the fp32 coefficients the kernels use
    z32 = float(torch.tensor(z, dtype=F32))
    names = ("lse", "loss_rows", "dlogits")
    ws = {n: Worst(f"{tag} {n}") for n in names}
    mut = [0.0] * len(mutants)
    s_ref = torch.zeros(4, dtype=F64, device=DEV)
    s_abs = torch.zeros(4, dtype=F64, device=DEV)
    s_bnd = torch.zeros(4, dtype=F64, device=DEV)
    cs_ref, cs_abs = cs_base.to(F64), cs_base.abs().to(F64)
    pad_ok, zero_max = True, 0.0
    for r0, r1 in _slabs(T, Vpad):
        h64 = h[r0:r1].to(F64)
        z_ = h64 @ W64 + b64
        delta = (K + 8) * UTC * (h64.abs() @ Wa + b64.abs())
        lse_ref = torch.logsumexp(z_, 1)
        eps_lse = delta.max(1).values + 5 * U * z_.abs().max(1).values + 2.0 ** -19 + (nt / 8 + 40) * U + \
            4 * U * lse_ref.abs()
        ws["lse"].add(lse[r0:r1], lse_ref, eps_lse, a=0.0, b=1.0)
        lab = labels[r0:r1].long()
        zl = z_.gather(1, lab[:, None])[:, 0]
        ce = lse_ref - zl
        zt = z32 * lse_ref ** 2
        loss = ce + zt
        eps_ce = eps_lse + delta.gather(1, lab[:, None])[:, 0] + 2 * U * ce.abs()
        lb = eps_ce + z32 * (2 * lse_ref.abs() * eps_lse + 3 * U * lse_ref ** 2) + 2 * U * loss.abs()
        ws["loss_rows"].add(lr[r0:r1], loss, lb, a=0.0, b=1.0)
        text = (torch.arange(r0, r1, device=DEV) % S) < TL - 1
        a = torch.where(text, a32[0], a32[1])
        for i, (v, b) in enumerate(((a * loss, a * lb), (torch.where(text, ce, 0.0), torch.where(text, eps_ce, 0.0)),
                                    (torch.where(text, 0.0, ce), torch.where(text, 0.0, eps_ce)),
                                    (zt, z32 * (2 * lse_ref.abs() * eps_lse + 3 * U * lse_ref ** 2)))):
            s_ref[i] += v.sum()
            s_abs[i] += v.abs().sum()
            s_bnd[i] += b.sum()
        p = torch.exp(z_ - lse_ref[:, None])
        onehot = torch.zeros_like(p).scatter_(1, lab[:, None], 1.0)
        c = a * (1 + 2 * z32 * lse_ref)
        ref = c[:, None] * p - a[:, None] * onehot
        eps_exp = 2.0 ** -21 + 5 * U * (z_.abs() + lse_ref.abs()[:, None]) + \
            2 * U * torch.log(c.abs().clamp_min(1e-300)).abs()[:, None]
        acc = (1.01 * c.abs()[:, None] * (delta + eps_lse[:, None] + eps_exp) + 2 * (a * z32 * eps_lse)[:, None]
               + 4 * U * c.abs()[:, None]) * p + U * a[:, None] * onehot
        ws["dlogits"].add(dl[r0:r1, :V], ref, acc, b=1.0, bf16_out=True, floor=2.0 ** -126)
        for i, q in enumerate(mutants):   # oracle.loss_weights.dlogits with the slab's row positions
            qa, _ = OW.row_coefficients(S, TL, IL, weights, Bg, q)
            am = qa.to(DEV)[torch.arange(r0, r1, device=DEV) % S]
            bad = am[:, None] * ((1 + q.z_grad_factor * z32 * lse_ref)[:, None] * p - onehot)
            mut[i] = max(mut[i], float64_bounds.worst_ratio(f"{tag} mutant", dl[r0:r1, :V], bad, acc, b=1.0,
                                                            bf16_out=True, floor=2.0 ** -126))
        zero_rows = a == 0
        if zero_rows.any():
            zero_max = max(zero_max, dl[r0:r1][zero_rows].float().abs().max().item())
        pad_ok &= bool((dl[r0:r1, V:] == 0).all())
        o64 = dl[r0:r1].to(F64)
        cs_ref, cs_abs = cs_ref + o64.sum(0), cs_abs + o64.abs().sum(0)
        del z_, delta, p, onehot, ref, acc, eps_exp, h64, o64
    worst = max(w.report() for w in ws.values())
    assert pad_ok, f"{tag}: padding columns of dlogits are not exactly 0"
    for i, name in enumerate(("weighted loss", "text CE", "image CE", "z-term")):
        worst = max(worst, check(f"{tag} sum {name}", sums[i:i + 1], (base[i:i + 1].to(F64) + s_ref[i:i + 1]),
                                 base[i:i + 1].abs().to(F64) + s_abs[i:i + 1], a=0.0, b=(T / 32 + 48) * U,
                                 floor=s_bnd[i].item() + 1e-30))
    worst = max(worst, check(f"{tag} dbias colsum", cs, cs_ref, cs_abs, a=0.0, b=(32 + T / 32 + 8) * U))
    for q, r in zip(mutants, mut):
        print(f"[loss-weights] {tag} mutant {q}: worst err/bound {r:.3g} (must exceed 1)")
        assert r > 1.0, f"{tag}: the kernel also satisfies the mutant oracle {q}"
    assert zero_max == 0.0, f"{tag}: a zero-weight class has non-zero dlogits ({zero_max})"
    return worst


def _labels(ops, cfg, T, S, g):
    tokens = synthetic_tokens(cfg, -(-T // S), g)
    labels = torch.empty_like(tokens)
    ops.shift_labels(tokens, labels, cfg["text_vocab_size"] + cfg["image_vocab_size"])
    return labels.view(-1)[:T].contiguous()


@pytest.mark.parametrize("config,T,weights,z", [
    ("dalle_example_b200", 40960, (1.0, 7.0), 1e-4),     # the bench shape
    ("dalle_coco_b200", 20480, (1.0, 7.0), 0.0),
    ("dalle_example_b200", 2 * 1280 + 333, (0.0, 1.0), 1e-4),   # ragged T, a zero-weight text class
    ("dalle_example_b200", 1280 + 77, (2.0, 0.0), 0.0),         # ragged T, a zero-weight image class
])
def test_weighted_cross_entropy_against_float64(ops, config, T, weights, z):
    from oracle import loss_weights as OW
    cfg = _config(config)
    K, V = cfg["n_embd"], cfg["text_vocab_size"] + cfg["image_vocab_size"] + 1
    Vpad, S, TL = (V + 63) // 64 * 64, 1280, cfg["text_seq_len"]
    g = _gen(T + K)
    h, W, bias, _, _ = ce_operands(T, K, V, Vpad, g)
    labels = _labels(ops, cfg, T, S, g)
    mutants = (OW.LossQuirks(text_rows_offset=0),) if weights == (1.0, 7.0) else ()
    run_weighted_ce(ops, f"{config} weighted CE T={T} w={weights} z={z}", T, K, V, Vpad, S, TL, labels=labels, h=h,
                    W=W, bias=bias, weights=weights, z=z, global_batch=max(1, T // S), mutants=mutants)


def test_rows_with_a_negative_coefficient(ops):
    """1 + 2 z lse <= 0 when lse < -1 / (2 z): a feature of value -40 on every other row meets a weight of 1 in every
    column, so those rows' lse is about -29 (z = 0.05: c' ~ -1.9); the other rows keep lse ~ 8.  Both mutants must
    fail here (the z factor matters at this z)."""
    from oracle import loss_weights as OW
    T, K, V, Vpad, S, TL = 2 * 1280 + 101, 128, 3001, 3008, 1280, 256
    g = _gen(5)
    h, W, bias, _, _ = ce_operands(T, K, V, Vpad, g)
    h[:, 0] = 0
    h[::2, 0] = -40.0
    W[0, :V] = 1.0
    labels = torch.randint(0, V, (T,), generator=g, device=DEV, dtype=I32)
    run_weighted_ce(ops, "negative rows T=2661", T, K, V, Vpad, S, TL, labels=labels, h=h, W=W, bias=bias,
                    weights=(1.0, 7.0), z=0.05, global_batch=2,
                    mutants=(OW.LossQuirks(text_rows_offset=0), OW.LossQuirks(z_grad_factor=1.0)))


def test_invalid_weights_descriptor_is_rejected(ops):
    import ctypes
    from dalle_mtf_b200 import lib as L
    lib, s = L.load(), torch.cuda.current_stream().cuda_stream
    x = torch.zeros(64, dtype=F32, device=DEV)
    e = L.GemmEpilogue()
    e.mode = L.EPI_CE_GRAD
    for bad in (L.make_ce_weights(0, 0, 1, 1, 0), L.make_ce_weights(10, 11, 1, 1, 0),
                L.make_ce_weights(10, 9, -1, 1, 0), L.make_ce_weights(10, 9, 1, float("nan"), 0),
                L.make_ce_weights(10, 9, 1, 1, -1e-4)):
        assert lib.db200_ce_finish_weighted(s, x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(),
                                            x.data_ptr(), 16, 1, ctypes.byref(bad), None, 0) != 0
        assert lib.db200_gemm_bf16_ce_weighted(s, x.data_ptr(), 0, 64, x.data_ptr(), 1, 64, x.data_ptr(), 64, 16, 64,
                                               64, ctypes.byref(e), ctypes.byref(bad)) != 0
    e.mode = L.EPI_STORE
    ok = L.make_ce_weights(10, 9, 1, 1, 0)
    assert lib.db200_gemm_bf16_ce_weighted(s, x.data_ptr(), 0, 64, x.data_ptr(), 1, 64, x.data_ptr(), 64, 16, 64, 64,
                                           ctypes.byref(e), ctypes.byref(ok)) != 0


# ------------------------------------------------------------------------------------------------------- engine
def relfro(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _engine(cfg, **kw):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    return DalleEngine(cfg.n_embd, cfg.n_layers, cfg.n_heads, cfg.text_vocab_size, cfg.image_vocab_size,
                       cfg.text_seq_len, cfg.image_seq_len, **kw)


def _step(eng, tok, grad_scale=1.0, global_batch=None, split=1):
    eng.zero_grads()
    mb = tok.shape[0] // split
    for i in range(split):
        eng.forward(tok[i * mb:(i + 1) * mb], global_batch=global_batch or tok.shape[0])
        eng.backward(grad_scale)
    torch.cuda.synchronize()
    return eng.grads.clone()


def test_dalle_example_weighted_step_with_caption_dropout_matches_the_oracle():
    """dalle_example geometry (d512 / L6 / H4 / S1280 / V50771), B = 2, captions dropped by caption_dropout's decisions,
    weights 1 : 7, z = 1e-4: loss within 1e-3, gradients no worse than 1.25 x the reference's bf16 policy + 1e-2."""
    from oracle import dalle as O
    from oracle import loss_weights as OW
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    cfg = O.DalleConfig(512, 6, 4, 50258, 512, 256, 1024)
    params = O.init_params(cfg, 17)
    g = torch.Generator().manual_seed(18)
    for k in params:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
    B, pad = 2, 50257
    text = torch.randint(0, pad, (B, 256), generator=g)
    text[:, 30:] = pad
    text[0] = pad                                      # sequence 0's caption dropped, sequence 1's kept
    tokens = O.assemble_tokens(text, torch.randint(0, 512, (B, 1024), generator=g), 50258)
    wz = ((1.0, 7.0), 1e-4)
    loss32, rows32, parts32, _, g32 = OW.loss_and_grads(params, tokens, cfg, *wz)
    _, _, _, _, g16 = OW.loss_and_grads(params, tokens, cfg, *wz, bf16=True)
    eng = _engine(cfg, loss_weights=wz[0], z_loss=wz[1])
    eng.load_params(params)
    tok = tokens.to(torch.int32).to(DEV)
    eng.zero_grads()
    acc = eng.forward(tok)
    eng.backward(1.0)
    torch.cuda.synchronize()
    loss = acc[0].item()
    assert abs(loss - loss32.item()) / loss32.item() <= 1e-3, (loss, loss32.item())
    assert relfro(eng._bufs["loss_rows"].view(B, -1), rows32) <= 5e-3
    scales = eng.loss_part_scales(B)
    for i in range(3):
        assert abs(acc[i + 1].item() * scales[i] - parts32[i].item()) <= 1e-3 * abs(parts32[i].item()), i
    grads = eng.export_params(eng.grads)
    worst = 0.0
    for k in g32:
        ee, er = relfro(grads[k], g32[k]), relfro(g16[k], g32[k])
        worst = max(worst, ee / (1.25 * er + 1e-2))
        assert ee <= 1.25 * er + 1e-2, (k, ee, er)
    assert (eng.G("wout")[:, eng.V:] == 0).all() and (eng.G("bout")[eng.V:] == 0).all()
    print(f"[loss-weights] EX weighted step: loss {loss:.6f} oracle {loss32.item():.6f}; worst gradient err / bound "
          f"{worst:.3f}")


def _small(seed=0):
    from oracle import dalle as O
    cfg = O.DalleConfig(256, 2, 2, 300, 60, 40, 88)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    tokens = torch.randint(0, cfg.total_tokens - 1, (4, cfg.seq_len), generator=g)
    tokens[:, 20:40] = 299
    return cfg, params, tokens.to(torch.int32).to(DEV)


def test_reference_ratio_equals_the_unweighted_step():
    cfg, params, tok = _small(1)
    T = tok.numel()
    plain = _engine(cfg)
    plain.load_params(params)
    plain.zero_grads()
    acc0 = plain.forward(tok).clone()
    plain.backward(1.0 / T)
    torch.cuda.synchronize()
    w = _engine(cfg, loss_weights=(cfg.text_seq_len - 1, cfg.image_seq_len + 1))
    w.load_params(params)
    gw = _step(w, tok)
    n = plain.n_params_padded
    assert relfro(gw[:n], plain.grads[:n]) < 1e-5
    assert abs(gw[w.aux_off].item() - acc0.item() / T) <= 1e-5 * acc0.item() / T
    assert torch.equal(w._bufs["loss_rows"], plain._bufs["loss_rows"])


def test_no_keys_launch_the_same_kernels(monkeypatch):
    """No weights and z_loss 0: the same calls (no ce_weights) and the same launch count as the plain engine."""
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops as O
    cfg, params, tok = _small(2)
    calls = []
    orig_gemm, orig_fin = O.gemm, O.ce_finish

    def spy_gemm(*a, **kw):
        calls.append(("gemm", kw.get("mode"), kw.get("ce_weights") is not None))
        return orig_gemm(*a, **kw)

    def spy_fin(*a, **kw):
        calls.append(("ce_finish",))
        return orig_fin(*a, **kw)
    monkeypatch.setattr(O, "gemm", spy_gemm)
    monkeypatch.setattr(O, "ce_finish", spy_fin)
    counts, lists = [], []
    for kw in ({}, {"z_loss": 0.0}, {"loss_weights": None, "z_loss": 0}):
        eng = _engine(cfg, **kw)
        eng.load_params(params)
        _step(eng, tok, 1.0 / tok.numel())
        calls.clear()
        n0 = L.launch_count()
        _step(eng, tok, 1.0 / tok.numel())
        counts.append(L.launch_count() - n0)
        lists.append(list(calls))
        assert not eng.weighted_loss
    assert len(set(counts)) == 1 and all(x == lists[0] for x in lists), counts
    assert not any(c[-1] for c in lists[0] if c[0] == "gemm")


def test_weighted_steps_are_bit_identical_and_micro_batching_matches():
    cfg, params, tok = _small(3)
    eng = _engine(cfg, loss_weights=(1.0, 7.0), z_loss=1e-4)
    eng.load_params(params)
    a, b = _step(eng, tok), _step(eng, tok)
    assert torch.equal(a, b)
    c = _step(eng, tok, split=2)
    n = eng.n_params_padded
    assert relfro(c[:n], a[:n]) < 1e-5
    assert torch.allclose(c[eng.aux_off:eng.aux_off + 4], a[eng.aux_off:eng.aux_off + 4], rtol=1e-5, atol=0)


@pytest.mark.parametrize("k", [4, 16])
def test_weighted_backward_with_reserved_sms(k):
    cfg, params, tok = _small(4)
    eng = _engine(cfg, loss_weights=(1.0, 7.0), z_loss=1e-4)
    eng.load_params(params)
    ref = _step(eng, tok)
    with float64_bounds.reserved_sms(k):
        got = _step(eng, tok)
    n = eng.n_params_padded
    assert relfro(got[:n], ref[:n]) < 1e-5
    assert torch.allclose(got[eng.aux_off:eng.aux_off + 4], ref[eng.aux_off:eng.aux_off + 4], rtol=1e-5, atol=0)


def _tiny_params(tmp_path, **extra):
    from collections import defaultdict
    vae = defaultdict(lambda: None, {"model_type": "vae", "num_tokens": 64, "convblocks": [[2, 64], [2, 64]],
                                     "dataset": {"image_size": 16}})
    p = defaultdict(lambda: None, {"model_type": "dalle", "dataset": {"image_size": 16}, "train_batch_size": 4,
                                   "eval_batch_size": 4, "n_embd": 256, "n_layers": 2, "n_heads": 2,
                                   "text_vocab_size": 300, "image_vocab_size": 64, "text_seq_len": 12, "lr": 2e-3,
                                   "train_steps": 100, "warmup_steps": 2, "bf_16": True, "mesh_shape": "data:1",
                                   "layout": "batch_dim:data", "model_path": str(tmp_path / "dalle"),
                                   "vae_params": vae, "vae_random_init": True, "seed": 5})
    p.update(extra)
    return p


def _batch():
    g = torch.Generator().manual_seed(3)
    return torch.rand(4, 16, 16, 3, generator=g) * 2 - 1, torch.randint(0, 299, (4, 12), generator=g)


WEIGHTED = {"text_loss_weight": 1, "image_loss_weight": 7, "z_loss": 1e-4, "caption_dropout": 0.5, "padding_id": 299}


def test_model_fn_train_and_eval_report_the_loss_and_its_parts(tmp_path):
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from oracle import loss_weights as OW
    img, cap = _batch()
    spec = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **WEIGHTED))
    n0 = len(spec.engine.grads)
    loss = spec.train_op(img, cap)
    assert spec.loss_scale == 1.0 and spec.loss_parts.shape == (3,) and spec.loss_parts.is_cuda
    parts = spec.loss_parts.tolist()
    total = loss.item()
    wt, wi = 1.0, 7.0
    assert len(spec.engine.grads) == n0 and parts[0] > 0 and parts[1] > 0 and parts[2] > 0
    # the loss is a weighted mean of per-class means of CE + z-term: between the smallest and largest class mean
    assert min(parts[0], parts[1]) < total < max(parts[0], parts[1]) + 10 * parts[2]
    S = spec.engine.S
    mb = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, tokens_per_mb_per_replica=2 * S, **WEIGHTED))
    assert tmp_path and mb.engine is not spec.engine
    assert math.isclose(mb.train_op(img, cap).item(), total, rel_tol=1e-5)
    assert torch.allclose(mb.loss_parts, spec.loss_parts, rtol=1e-5)
    # eval: the forward's rows against the oracle formula on the engine's own logits
    ev = dalle_model_fn(img, cap, "eval", _tiny_params(tmp_path, **WEIGHTED))
    el = ev.eval_op(img, cap).item()
    eng = ev.engine
    toks = ev.assemble(img, cap).clone()
    logits = eng.logits(toks).double().cpu()
    labels = torch.cat([toks[:, 1:], torch.full_like(toks[:, :1], eng.eos_token_id)], 1).long().cpu()
    ref, rows, rparts = OW.weighted_loss(logits, labels, 12, eng.image_seq_len, (wt, wi), 1e-4)
    assert math.isclose(el, ref.item(), rel_tol=1e-4), (el, ref.item())
    for a, b in zip(ev.loss_parts.tolist(), rparts):
        assert math.isclose(a, b.item(), rel_tol=1e-4, abs_tol=1e-7)
    ev.eval_op(img, cap)
    assert relfro(eng._bufs["loss_rows"].view(4, -1), rows) < 1e-4
    # without the keys there are no parts and the loss is the plain mean
    plain = dalle_model_fn(img, cap, "eval", _tiny_params(tmp_path))
    plain.eval_op(img, cap)
    assert plain.loss_parts is None and plain.loss_scale != 1.0


def test_dalle_class_forward_reports_the_parts_and_loss_batch():
    from dalle_mtf_b200.models import DALLE
    from oracle import loss_weights as OW
    m = DALLE(256, text_vocab_size=300, image_vocab_size=60, text_seq_len=40, image_seq_len=88, n_layers=1, n_heads=2,
              mode="eval", params={"text_loss_weight": 1, "image_loss_weight": 7, "z_loss": 1e-3})
    g = torch.Generator().manual_seed(9)
    tokens = torch.randint(0, 360, (2, 128), generator=g)
    loss, loss_batch = m.forward({"tokens": tokens})
    logits = m.engine.logits(tokens.to(torch.int32).to(DEV)).double().cpu()
    labels = torch.cat([tokens[:, 1:], torch.full_like(tokens[:, :1], m.eos_token_id)], 1)
    ref, rows, parts = OW.weighted_loss(logits, labels, 40, 88, (1.0, 7.0), 1e-3)
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-4)
    assert relfro(loss_batch, rows) < 1e-4
    for a, b in zip(m.loss_parts.tolist(), parts):
        assert math.isclose(a, b.item(), rel_tol=1e-4)


def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dp_worker(rank, world, port, out):
    os.environ.update({"RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank),
                       "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)})
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.dist import DataParallel
    dp = DataParallel().init()
    dev = torch.device("cuda", rank)
    args = (256, 2, 2, 500, 64, 24, 40)
    kw = dict(device=dev, loss_weights=(1.0, 7.0), z_loss=1e-4)
    tokens = torch.randint(0, 500 + 64, (4, 64), generator=torch.Generator().manual_seed(0), dtype=torch.int32)
    eng = DalleEngine(*args, **kw)
    eng.init_params(seed=7)
    start, per = dp.shard(4)
    eng.zero_grads()
    eng.forward(tokens[start:start + per].to(dev), global_batch=4)
    eng.backward(1.0, on_bucket_ready=dp.make_bucket_hook(eng.grads))
    dp.wait()
    ref = DalleEngine(*args, **kw)
    ref.init_params(seed=7)
    ref.zero_grads()
    ref.forward(tokens.to(dev), global_batch=4)
    ref.backward(1.0)
    torch.cuda.synchronize()
    n = eng.n_params_padded
    gerr = ((eng.grads[:n] - ref.grads[:n]).norm() / ref.grads[:n].norm()).item()
    aux = (eng.grads[eng.aux_off:eng.aux_off + 4].tolist(), ref.grads[ref.aux_off:ref.aux_off + 4].tolist())
    dp.barrier()
    out.put((rank, gerr, aux))
    dp.shutdown()


def test_two_rank_weighted_step_equals_one_rank():
    """Rank r of 2 processes sequences [2r, 2r + 2) with the coefficients of the global batch of 4; the all-reduced
    gradients and the four sums equal the 1-rank step on the 4 sequences."""
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(out.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for rank, gerr, (got, ref) in res:
        assert gerr < 2e-3, res
        assert all(math.isclose(a, b, rel_tol=1e-5, abs_tol=1e-12) for a, b in zip(got, ref)), res
