"""GPU tests of local (sliding-window) attention: query i attends to keys (i - r, i] (src/dalle_mtf/models.py:257-273).

Kernels against float64 with the bounds of the causal kernels (test_dalle_kernels_gpu.py's module docstring; the
reference here masks the band instead of the lower triangle), their equality with the causal entry points at r >= S,
and a window check: on inputs with constant logits the lse of every row is log(#visible keys), so the kernel's output
must fail the same comparison against the oracle at r - 1 and at r + 1.  Then the engine against the oracle with mixed
layer types (fp32 and the reference bf16 policy, recompute_grad off and on, with and without dropout), the decoder
(db200_attn_decode_local* against float64, graph replay, greedy generation, prefill, guidance) and dalle_model_fn.
"""
import functools
import math

import pytest
import torch

import float64_bounds
from float64_bounds import DEV, U, UTC, nan_like

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
TAG = "local-attention"
UBF = 2.0 ** -8
worst = functools.partial(float64_bounds.worst_ratio)


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def relfro(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _qkv(B, S, H, dh, g):
    qkv = torch.randn(B, S, 3, H, dh, generator=g, device=DEV)
    qkv[:, :, :2] *= 1.3 * dh ** -0.25
    return qkv.to(BF16), torch.randn(B, S, H, dh, generator=g, device=DEV).to(BF16)


# ------------------------------------------------------------------------------------------------------- kernels
def band(S, r):
    i = torch.arange(S, device=DEV)[:, None]
    j = torch.arange(S, device=DEV)[None, :]
    return (j <= i) & (j > i - r)


def local_reference(q, k, v, do, o, scale, r):
    """float64 local attention forward / backward, the |.| graphs and the bounds of the causal kernels' test on
    [B, S, H, dh] operands (o: the kernel's own output, which delta uses as the kernel does).  do = None: the forward
    only (O and lse; b_bwd is None)."""
    q, k, v = (t.to(F64).permute(0, 2, 1, 3) for t in (q, k, v))
    S, dh = q.shape[2], q.shape[3]
    mask = band(S, r)
    s = (scale * q @ k.transpose(-1, -2)).masked_fill(~mask, -math.inf)
    sa = scale * q.abs() @ k.abs().transpose(-1, -2)
    lse = torch.logsumexp(s, -1)
    P = torch.exp(s - lse[..., None])
    m = s.max(-1).values
    eps_s = ((dh + 8) * UTC * sa + 3 * U * (s.abs().masked_fill(~mask, 0) + m.abs()[..., None])).masked_fill(~mask, 0)
    eps_row = eps_s.max(-1).values
    nblk = -(-S // 64)
    eps_lse = eps_row + (S + 32) * U + (nblk + 4) * 2.0 ** -21 + 2 * U * lse.abs()
    out = {"O": (P @ v, P @ v.abs()), "lse": (lse, eps_lse)}
    b_fwd = UBF + 2 * eps_row + (2 * nblk + 2) * 2.0 ** -21 + (2 * S + 2 * nblk + 32) * UTC
    b_bwd = None
    if do is not None:
        do, o = do.to(F64).permute(0, 2, 1, 3), o.to(F64).permute(0, 2, 1, 3)
        dP, dPa = do @ v.transpose(-1, -2), do.abs() @ v.abs().transpose(-1, -2)
        delta, deltaa = (do * o).sum(-1, keepdim=True), (do * o).abs().sum(-1, keepdim=True)
        dS, dSa = P * (dP - delta), P * (dPa + deltaa)
        out["dQ"] = (scale * dS @ k, scale * dSa @ k.abs())
        out["dK"] = (scale * dS.transpose(-1, -2) @ q, scale * dSa.transpose(-1, -2) @ q.abs())
        out["dV"] = (P.transpose(-1, -2) @ do, P.transpose(-1, -2) @ do.abs())
        b_bwd = (eps_s + eps_lse[..., None]).masked_fill(~mask, 0).max().item() + 2.0 ** -20 + UBF + \
            (S + dh + 24) * UTC
    out = {n:(x.permute(0, 2, 1, 3) if x.dim() == 4 else x, a.permute(0, 2, 1, 3) if a.dim() == 4 else a)
           for n, (x, a) in out.items()}
    return out, b_fwd.permute(0, 2, 1)[..., None], b_bwd


def run_local(ops, qkv, dout, r, scale=1.0):
    B, S, _, H, dh = qkv.shape
    out, lse = nan_like((B, S, H, dh), BF16), nan_like((B, H, S), F32)
    ops.attn_fwd(qkv, out, lse, B, S, H, dh, scale, radius=r)
    dqkv = nan_like((B, S, 3, H, dh), BF16)
    ops.attn_bwd(qkv, out, dout, lse, torch.zeros(1, device=DEV), nan_like((B, H, S), F32), dqkv, B, S, H, dh, scale,
                 radius=r)
    return out, lse, dqkv


def ratios(qkv, dout, out, lse, dqkv, r, scale=1.0):
    """{output: worst err/bound} of the kernel's outputs against the float64 local attention of radius r."""
    refs, b_fwd, b_bwd = local_reference(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], dout, out, scale, r)
    res = {"O": worst("O", out, *refs["O"], b=b_fwd, bf16_out=True, floor=2.0 ** -120),
           "lse": worst("lse", lse, refs["lse"][0], refs["lse"][1], a=0.0, b=1.0)}
    for i, n in enumerate(("dQ", "dK", "dV")):
        res[n] = worst(n, dqkv[:, :, i], *refs[n], b=b_bwd, bf16_out=True, floor=2.0 ** -120)
    return res


S_CASES = (1280, 1000)     # the dalle_example length and a ragged one (not a multiple of 64)


def _radii(S):
    return (1, 63, 64, 65, 256, S - 1, S)


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("S", S_CASES)
def test_local_kernels_against_float64(ops, S, dh):
    B, H = 2, 2
    for r in _radii(S):
        qkv, dout = _qkv(B, S, H, dh, _gen(S + dh + r))
        out, lse, dqkv = run_local(ops, qkv, dout, r)
        for n, v in ratios(qkv, dout, out, lse, dqkv, r).items():
            float64_bounds.report(f"local S={S} dh={dh} r={r} {n}", v, TAG)


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("S", S_CASES)
def test_window_edges_are_exact(ops, S, dh):
    """q = 0: every visible key has logit 0, so lse_i = log(min(i + 1, r)) and O_i is the mean of the visible v.  The
    kernel passes against the oracle at r and fails at r - 1 and at r + 1 (the radius the kernel ran is pinned)."""
    B, H = 1, 2
    for r in _radii(S):
        qkv, dout = _qkv(B, S, H, dh, _gen(S * dh + r))
        qkv[:, :, 0] = 0
        out, lse, dqkv = run_local(ops, qkv, dout, r)
        assert max(ratios(qkv, dout, out, lse, dqkv, r).values()) < 1.0, r
        rows = torch.arange(S, device=DEV, dtype=F64)
        assert (lse.to(F64) - torch.log(torch.clamp(rows + 1, max=r))).abs().max() < 1e-5
        for wrong in (r - 1, r + 1):
            if 1 <= wrong and min(wrong, S) != min(r, S):
                got = max(ratios(qkv, dout, out, lse, dqkv, wrong).values())
                print(f"[{TAG}] S={S} dh={dh} kernel r={r} against oracle r={wrong}: worst err/bound {got:.1f}")
                assert got > 1.0, (r, wrong)


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("S", S_CASES)
def test_radius_at_least_s_equals_the_causal_entry_points(ops, S, dh):
    B, H = 2, 2
    qkv, dout = _qkv(B, S, H, dh, _gen(S - dh))
    out0, lse0 = nan_like((B, S, H, dh), BF16), nan_like((B, H, S), F32)
    ops.attn_fwd(qkv, out0, lse0, B, S, H, dh, 1.0)
    dqkv0 = nan_like((B, S, 3, H, dh), BF16)
    ops.attn_bwd(qkv, out0, dout, lse0, torch.zeros(1, device=DEV), nan_like((B, H, S), F32), dqkv0, B, S, H, dh, 1.0)
    for r in (S, S + 1, 4 * S):
        out, lse, dqkv = run_local(ops, qkv, dout, r)
        assert torch.equal(out, out0) and torch.equal(lse, lse0) and torch.equal(dqkv, dqkv0), r


def test_invalid_radius_is_rejected(ops):
    from dalle_mtf_b200 import lib as L
    lib = L.load()
    B, S, H, dh = 1, 64, 1, 64
    qkv = torch.zeros(B, S, 3, H, dh, dtype=BF16, device=DEV)
    out, lse = torch.zeros(B, S, H, dh, dtype=BF16, device=DEV), torch.zeros(B, H, S, device=DEV)
    s = L.stream_ptr()
    for r in (0, -1):
        assert lib.db200_attn_local_fwd(s, qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, S, H, dh, r, 1.0) != 0
        assert lib.db200_attn_local_bwd(s, qkv.data_ptr(), out.data_ptr(), out.data_ptr(), lse.data_ptr(), None,
                                        lse.data_ptr(), qkv.data_ptr(), B, S, H, dh, r, 1.0) != 0
        kc = torch.zeros(B, S, H, dh, dtype=BF16, device=DEV)
        step = torch.zeros(B, 3, H, dh, dtype=BF16, device=DEV)
        pos = torch.zeros(1, dtype=I32, device=DEV)
        assert lib.db200_attn_decode_local(s, step.data_ptr(), kc.data_ptr(), kc.data_ptr(), out.data_ptr(), B, S, H,
                                           dh, 3, r, 1.0) != 0
        assert lib.db200_attn_decode_local_dev(s, step.data_ptr(), kc.data_ptr(), kc.data_ptr(), out.data_ptr(), B, S,
                                               H, dh, pos.data_ptr(), r, 1.0) != 0
    with pytest.raises(L.DB200Error):
        ops.attn_fwd(qkv, out, lse, B, S, H, dh, 1.0, radius=0)
    with pytest.raises(L.DB200Error):
        ops.attn_fwd(qkv, out, lse, B, S, H, dh, 1.0, radius=4, dropout=L.make_dropout(0.1, 0, 0, 2, 0))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- decode
def decode_reference(q, k, v, scale):
    """test_dalle_kernels_gpu.py's attn_decode bound over the window's keys k, v [B, n, H, dh]."""
    dh = q.shape[-1]
    q = q.to(F64)
    k, v = k.to(F64).permute(0, 2, 1, 3), v.to(F64).permute(0, 2, 1, 3)
    s = scale * (k @ q[..., None])[..., 0]
    sa = abs(scale) * (k.abs() @ q.abs()[..., None])[..., 0]
    P = torch.softmax(s, -1)
    eps = ((dh + 8) * U * sa + 3 * U * (s.abs() + s.max(-1, keepdim=True).values.abs())).max(-1).values
    b = UBF + 2 * eps + 2.0 ** -20 + (k.shape[2] / 8 + 40) * U
    return (P[..., None, :] @ v)[..., 0, :], (P[..., None, :] @ v.abs())[..., 0, :], b[..., None]


@pytest.mark.parametrize("dh", [64, 128])
def test_attn_decode_local_against_float64_around_the_window_edge(ops, dh):
    B, S, H = 4, 1280, 512 // dh
    g = _gen(dh + 11)
    for r in (64, 256):
        for pos in (0, r - 2, r - 1, r, r + 1, S - 1):
            kc = (torch.randn(B, S, H, dh, generator=g, device=DEV) * 1.3 * dh ** -0.25).to(BF16)
            vc = torch.randn(B, S, H, dh, generator=g, device=DEV).to(BF16)
            step = torch.randn(B, 3, H, dh, generator=g, device=DEV)
            step[:, :2] *= 1.3 * dh ** -0.25
            step = step.to(BF16)
            kc2, vc2 = kc.clone(), vc.clone()
            out = nan_like((B, H, dh), BF16)
            ops.attn_decode(step, kc, vc, out, pos, 1.0, radius=r)
            assert torch.equal(kc[:, pos], step[:, 1]) and torch.equal(vc[:, pos], step[:, 2])
            lo = max(0, pos - r + 1)
            ref, absref, b = decode_reference(step[:, 0], kc[:, lo:pos + 1], vc[:, lo:pos + 1], 1.0)
            float64_bounds.check(f"attn_decode_local dh={dh} r={r} pos={pos}", out, ref, absref, b=b, bf16_out=True,
                                 tag=TAG)
            # the device-position variant computes the same, and r >= S is the global kernel
            pos_dev = torch.full((1,), pos, dtype=I32, device=DEV)
            out_dev = nan_like((B, H, dh), BF16)
            ops.attn_decode_dev(step, kc2, vc2, out_dev, pos_dev, 1.0, radius=r)
            assert torch.equal(out_dev, out) and torch.equal(kc2, kc)
            og, ol = nan_like((B, H, dh), BF16), nan_like((B, H, dh), BF16)
            ops.attn_decode(step, kc2, vc2, og, pos, 1.0)
            ops.attn_decode(step, kc2, vc2, ol, pos, 1.0, radius=S)
            assert torch.equal(og, ol)


# ------------------------------------------------------------------------------------------------------- engine
RATES = (0.1, 0.2, 0.15)
# d, layers, H, text vocab, image vocab, text len, image len, B, layer types, radius
CASES = [(256, 2, 2, 1000, 100, 40, 24, 3, ("local", "global"), 16),
         (256, 3, 4, 1000, 100, 100, 60, 2, ("global", "local", "local"), 37),
         (512, 2, 4, 3000, 512, 200, 100, 2, ("local", "global"), 100)]


def _case(d, Ly, H, tv, iv, ts, isl, B, types, radius, recompute=False, rates=(0.0, 0.0, 0.0), dseed=0, seed=0):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    from oracle import dalle_local as OL
    cfg = OL.LocalConfig(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=radius)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if k.endswith("/g"):
            params[k] = 1 + torch.randn(params[k].shape, generator=g) * 0.05
    tokens = torch.randint(0, cfg.total_tokens - 1, (B, cfg.seq_len), generator=g)
    eng = DalleEngine(d, Ly, H, tv, iv, ts, isl, recompute_grad=recompute, dropout=rates, dropout_seed=dseed,
                      attention_types=types, local_attention_radius=radius)
    eng.load_params(params)
    return cfg, params, tokens, eng


@pytest.mark.parametrize("rates", [(0.0, 0.0, 0.0), RATES], ids=["no-dropout", "dropout"])
@pytest.mark.parametrize("case", CASES)
def test_mixed_engine_matches_the_oracle_recompute_off_and_on(case, rates):
    from oracle import dalle_dropout as D
    from oracle import dalle_local as OL
    step, row0, dseed = 6, 1, 11
    spec = (rates, dseed, step, row0)
    cfg, params, tokens, _ = _case(*case, rates=rates, dseed=dseed)
    loss32, _, logits32, g32 = OL.loss_and_grads(params, tokens, cfg, spec, bf16=False)
    _, _, logits16, g16 = OL.loss_and_grads(params, tokens, cfg, spec, bf16=True)
    tok = tokens.to(I32).cuda()
    T = tokens.numel()
    by_mode = []
    for recompute in (False, True):
        _, _, _, eng = _case(*case, recompute=recompute, rates=rates, dseed=dseed)
        eng.zero_grads()
        acc = eng.forward(tok, step=step, row0=row0)
        eng.backward(1.0 / T)
        torch.cuda.synchronize()
        assert abs(acc.item() / T - loss32.item()) / loss32.item() < 2e-3, recompute
        grads = eng.export_params(eng.grads)
        for k in g32:
            e_engine, e_ref = relfro(grads[k], g32[k]), relfro(g16[k], g32[k])
            assert e_engine <= 1.25 * e_ref + 1e-2, (recompute, k, e_engine, e_ref)
        by_mode.append(eng.grads.clone())
        if not any(rates):
            lg = eng.logits(tok)
            assert relfro(lg, logits32) <= 1.25 * relfro(logits16, logits32) + 1e-2
    assert torch.equal(by_mode[0], by_mode[1])
    # the local layers differ from global ones: the same weights without attention_types give another loss
    from oracle import dalle as O
    gcfg = O.DalleConfig(*case[:7])
    assert abs(D.loss_and_grads(params, tokens, gcfg, spec)[0].item() - loss32.item()) > 1e-4


def _three_steps(types, radius=16, rates=RATES):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    eng = DalleEngine(256, 2, 2, 500, 64, 64, 64, dropout=rates, dropout_seed=1, attention_types=types,
                      local_attention_radius=radius)
    eng.init_params(3)
    tok = torch.randint(0, 40, (4, eng.S), generator=torch.Generator(device=DEV).manual_seed(7), device=DEV, dtype=I32)
    out = []
    for s in range(3):
        eng.zero_grads()
        acc = eng.forward(tok, step=s)
        eng.backward(1.0 / tok.numel())
        out.append((acc.clone(), eng.grads.clone()))
        eng.optimizer_step(1e-3)
    torch.cuda.synchronize()
    return out, eng.master.clone()


def test_mixed_training_is_bitwise_reproducible():
    (a, pa), (b, pb) = _three_steps(["local", "global"]), _three_steps(["local", "global"])
    for (la, ga), (lb, gb) in zip(a, b):
        assert torch.isfinite(ga).all() and torch.equal(la, lb) and torch.equal(ga, gb)
    assert torch.equal(pa, pb)
    assert not torch.equal(_three_steps(["global", "global"])[1], pa)


def test_engine_without_attention_types_launches_the_causal_kernels(monkeypatch):
    """attention_types None (and an explicit all-global list) call the causal entry points only, with the same
    results; a mixed engine calls the local ones for its local layers."""
    from dalle_mtf_b200 import lib as L
    lib = L.load()
    seen = []
    for name in ("db200_attn_causal_fwd", "db200_attn_causal_fwd_ex", "db200_attn_causal_bwd",
                 "db200_attn_causal_bwd_ex", "db200_attn_local_fwd", "db200_attn_local_bwd"):
        fn = getattr(lib, name)
        monkeypatch.setattr(lib, name, lambda *a, _fn=fn, _n=name: (seen.append(_n), _fn(*a))[1])

    def run(types, rates=RATES):
        seen.clear()
        out, p = _three_steps(types, rates=rates)
        return list(seen), out, p

    calls, out0, p0 = run(None)
    assert set(calls) == {"db200_attn_causal_fwd_ex", "db200_attn_causal_bwd_ex"}
    calls1, out1, p1 = run(["global", "global"])
    assert calls1 == calls and torch.equal(p0, p1) and all(torch.equal(x[1], y[1]) for x, y in zip(out0, out1))
    calls, _, _ = run(None, rates=(0.0, 0.0, 0.0))
    assert set(calls) == {"db200_attn_causal_fwd", "db200_attn_causal_bwd"}
    calls, _, _ = run(["global", "local"])
    assert calls.count("db200_attn_local_fwd") == 3 and calls.count("db200_attn_local_bwd") == 3
    assert calls.count("db200_attn_causal_fwd_ex") == 3


# ------------------------------------------------------------------------------------------------------- generation
GEN = [(256, 2, 2, 300, 64, 24, 40, 3, ("local", "global"), 11, 29),
       (256, 3, 4, 500, 100, 70, 90, 2, ("global", "local", "local"), 45, 77)]


def _sharp(d, Ly, H, tv, iv, ts, isl, types, radius):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    from oracle import dalle_local as OL
    cfg = OL.LocalConfig(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=radius)
    params = O.init_params(cfg, 3)
    g = torch.Generator().manual_seed(9)
    for k in params:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if "wte" in k or "wout" in k or k.endswith("kernel"):
            params[k] = params[k] * 4
    eng = DalleEngine(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=radius)
    eng.load_params(params)
    return eng, params, cfg


@pytest.mark.parametrize("d,Ly,H,tv,iv,ts,isl,B,types,radius,P", GEN)
def test_mixed_generation_follows_the_full_forward_pass(d, Ly, H, tv, iv, ts, isl, B, types, radius, P):
    from dalle_mtf_b200.sampling import DalleSampler
    from oracle import dalle_local as OL
    eng, params, cfg = _sharp(d, Ly, H, tv, iv, ts, isl, types, radius)
    g = torch.Generator().manual_seed(4)
    text = torch.randint(0, tv, (B, ts), generator=g).to(I32).cuda()
    smp = DalleSampler(eng)
    toks, step_logits = smp.generate(text, temperature=0, return_logits=True)
    S = ts + isl
    img = toks[:, ts:]
    assert (img >= tv).all() and (img < tv + iv).all()
    full = eng.logits(toks)
    dec = torch.stack(step_logits, 1)
    assert relfro(dec, full[:, :S - 1]) < 2e-2
    rng = full[:, ts - 1:S - 1, tv:tv + iv]
    top2 = rng.topk(2, -1).values
    clear = (top2[..., 0] - top2[..., 1]) > 0.05 * rng.abs().max()
    same = (rng.argmax(-1) + tv) == img
    assert (same | ~clear).all() and clear.float().mean() > 0.2 and same.float().mean() > 0.8
    _, _, logits32, _ = OL.loss_and_grads(params, toks.cpu().long(), cfg, bf16=False)
    assert relfro(dec, logits32[:, :S - 1]) < 3e-2
    # graph replay: the same tokens as the eager loop
    assert torch.equal(smp.generate_graphed(text, temperature=0.0), toks)
    # prefill: the caches of the teacher-forced decode and the logits of position P, within test_prefill_gpu's bounds
    kc = [torch.zeros_like(c) for c in smp.kc]
    vc = [torch.zeros_like(c) for c in smp.vc]
    smp.generate(text, temperature=0)
    logits = eng.prefill(toks[:, :P].contiguous(), kc, vc).clone()
    assert torch.equal(kc[0][:, :P], smp.kc[0][:, :P]) and torch.equal(vc[0][:, :P], smp.vc[0][:, :P])
    for i in range(1, Ly):
        assert relfro(kc[i][:, :P], smp.kc[i][:, :P]) <= 1e-2, i
        assert relfro(vc[i][:, :P], smp.vc[i][:, :P]) <= 1e-2, i
    assert relfro(logits[:, :eng.V], full[:, P - 1]) < 2e-2
    assert relfro(logits[:, :eng.V], logits32[:, P - 1]) < 3e-2
    # completion from the prefill continues greedily like the full generation
    out = smp.complete(text, toks[:, ts:P] - tv, temperature=0)
    assert torch.equal(out[:, :P], toks[:, :P]) and (out[:, P:] >= tv).all() and (out[:, P:] < tv + iv).all()


def test_guided_generation_runs_on_a_mixed_model():
    from dalle_mtf_b200.sampling import DalleSampler
    eng, _, _ = _sharp(256, 2, 2, 300, 64, 24, 40, ("local", "global"), 11)
    smp = DalleSampler(eng)
    text = torch.randint(0, 299, (3, 24), generator=torch.Generator().manual_seed(2)).to(I32).cuda()
    eager = smp.generate(text, temperature=0.0, guidance_scale=3.0)
    graphed = smp.generate_graphed(text, temperature=0.0, guidance_scale=3.0)
    assert torch.equal(eager, graphed) and torch.equal(eager[:, :24], text)
    assert ((eager[:, 24:] >= 300) & (eager[:, 24:] < 364)).all()
    assert not torch.equal(eager, smp.generate(text, temperature=0.0))
    torch.manual_seed(0)
    a = smp.complete(text, samples_per_prompt=2, temperature=1.0, guidance_scale=3.0, top_k=8)
    torch.manual_seed(0)
    b = smp.complete(text, samples_per_prompt=2, temperature=1.0, guidance_scale=3.0, top_k=8)
    assert torch.equal(a, b) and a.shape == (6, 64) and ((a[:, 24:] >= 300) & (a[:, 24:] < 364)).all()


# ------------------------------------------------------------------------------------------------------- model_fn
def test_model_fn_trains_and_evaluates_with_local_layers(tmp_path):
    from collections import defaultdict
    from dalle_mtf_b200.model_fns import dalle_model_fn
    vae = defaultdict(lambda: None, {"model_type": "vae", "num_tokens": 64, "convblocks": [[2, 64], [2, 64]],
                                     "dataset": {"image_size": 16}})

    def params(**extra):
        p = defaultdict(lambda: None, {"model_type": "dalle", "dataset": {"image_size": 16}, "train_batch_size": 4,
                                       "eval_batch_size": 4, "n_embd": 256, "n_layers": 2, "n_heads": 2,
                                       "text_vocab_size": 300, "image_vocab_size": 64, "text_seq_len": 12, "lr": 2e-3,
                                       "train_steps": 100, "warmup_steps": 2, "bf_16": True, "mesh_shape": "data:1",
                                       "layout": "batch_dim:data", "model_path": str(tmp_path / "dalle"),
                                       "vae_params": vae, "vae_random_init": True, "seed": 5,
                                       "attention_dropout": 0.1, "residual_dropout": 0.1})
        p.update(extra)
        return p

    g = torch.Generator().manual_seed(3)
    img, cap = torch.rand(4, 16, 16, 3, generator=g) * 2 - 1, torch.randint(0, 299, (4, 12), generator=g)
    local = dict(attention_types=[[["global", "local"], 1]], local_attention_radius=5)
    spec = dalle_model_fn(img, cap, "train", params(**local))
    assert spec.engine.radii == [None, 5]
    losses = [spec.train_op(img, cap).item() * spec.loss_scale for _ in range(2)]
    ev = spec.eval_op(img, cap).item() * spec.loss_scale
    assert all(math.isfinite(x) and 0 < x < 20 for x in losses + [ev])
    plain = dalle_model_fn(img, cap, "eval", params())
    assert plain.engine.radii == [None, None]
    ev_local = dalle_model_fn(img, cap, "eval", params(**local)).eval_op(img, cap).item()
    assert ev_local != plain.eval_op(img, cap).item()
    with pytest.raises(ValueError, match="attention_types"):
        dalle_model_fn(img, cap, "train", params(attention_types=[[["local"], 3]]))
