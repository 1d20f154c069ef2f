"""GPU tests of axial (row and column) attention layers (dalle_mtf_b200/csrc/attn_fa.cu, AXIAL; decode.cu).

Text length TL, a W x W image grid: text queries are causal; an image query sees every text key plus its own grid row
at columns <= c (row layers, axis 0) or its own grid column at rows <= r (column layers, axis 1).  The kernels are
checked against float64 with the bounds of the causal kernels (test_local_attention_gpu.py's local_reference with the
axial mask in place of the band) at geometries that break tile assumptions: segments that straddle 64-row tiles,
W > 64, TL not a multiple of 64, W = 1.  A mask test runs q = 0 (every visible key has logit 0, so lse counts the
visible keys) and must fail against an oracle whose segment is shifted by one key.  Then prompt prefills at ragged
lengths, the decode kernels (host and device position, bit for bit), an engine with mixed layer types against
tests/axial_oracle.py, the attention calls it makes, generation and dalle_model_fn.  The module prints its wall time and
peak device memory.
"""
import math
import time

import pytest
import torch

import axial_oracle as OA
import float64_bounds
from float64_bounds import DEV, U, UTC, nan_like
from test_local_attention_gpu import RATES, UBF, _gen, _qkv, decode_reference, relfro, worst

pytestmark = pytest.mark.gpu

F64, F32, BF16, I32 = torch.float64, torch.float32, torch.bfloat16, torch.int32
TAG = "axial-attention"
NAMES = ("axial_row", "axial_col")


@pytest.fixture(scope="module", autouse=True)
def _module_cost():
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n[{TAG}] module wall time {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB on {torch.cuda.get_device_name()}")


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


# ------------------------------------------------------------------------------------------------------- kernels
def visible(S, TL, W, axis, shift=0):
    return ~OA.axial_hidden(S, TL, W, axis, shift).to(DEV)


def masked_reference(q, k, v, do, o, scale, mask):
    """test_local_attention_gpu.local_reference with an arbitrary [S,S] visibility mask (every row sees a key).
    do = None: the forward only (O and lse; b_bwd is None)."""
    q, k, v = (t.to(F64).permute(0, 2, 1, 3) for t in (q, k, v))
    S, dh = q.shape[2], q.shape[3]
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
    if do is None:
        out = {n: (x.permute(0, 2, 1, 3) if x.dim() == 4 else x, a.permute(0, 2, 1, 3) if a.dim() == 4 else a)
               for n, (x, a) in out.items()}
        return out, b_fwd.permute(0, 2, 1)[..., None], None
    do, o = do.to(F64).permute(0, 2, 1, 3), o.to(F64).permute(0, 2, 1, 3)
    dP, dPa = do @ v.transpose(-1, -2), do.abs() @ v.abs().transpose(-1, -2)
    delta, deltaa = (do * o).sum(-1, keepdim=True), (do * o).abs().sum(-1, keepdim=True)
    dS, dSa = P * (dP - delta), P * (dPa + deltaa)
    out["dQ"] = (scale * dS @ k, scale * dSa @ k.abs())
    out["dK"] = (scale * dS.transpose(-1, -2) @ q, scale * dSa.transpose(-1, -2) @ q.abs())
    out["dV"] = (P.transpose(-1, -2) @ do, P.transpose(-1, -2) @ do.abs())
    b_bwd = (eps_s + eps_lse[..., None]).masked_fill(~mask, 0).max().item() + 2.0 ** -20 + UBF + (S + dh + 24) * UTC
    out = {n: (x.permute(0, 2, 1, 3) if x.dim() == 4 else x, a.permute(0, 2, 1, 3) if a.dim() == 4 else a)
           for n, (x, a) in out.items()}
    return out, b_fwd.permute(0, 2, 1)[..., None], b_bwd


def run_axial(ops, qkv, dout, geom, scale=1.0):
    B, S, _, H, dh = qkv.shape
    out, lse = nan_like((B, S, H, dh), BF16), nan_like((B, H, S), F32)
    ops.attn_fwd(qkv, out, lse, B, S, H, dh, scale, axial=geom)
    dqkv = nan_like((B, S, 3, H, dh), BF16)
    ops.attn_bwd(qkv, out, dout, lse, torch.zeros(1, device=DEV), nan_like((B, H, S), F32), dqkv, B, S, H, dh, scale,
                 axial=geom)
    return out, lse, dqkv


def ratios(qkv, dout, out, lse, dqkv, mask, scale=1.0):
    refs, b_fwd, b_bwd = masked_reference(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], dout, out, scale, mask)
    res = {"O": worst("O", out, *refs["O"], b=b_fwd, bf16_out=True, floor=2.0 ** -120),
           "lse": worst("lse", lse, refs["lse"][0], refs["lse"][1], a=0.0, b=1.0)}
    for i, n in enumerate(("dQ", "dK", "dV")):
        res[n] = worst(n, dqkv[:, :, i], *refs[n], b=b_bwd, bf16_out=True, floor=2.0 ** -120)
    return res


# (TL, W, B, H): the dalle_example grid; W not dividing 64 and TL not a multiple of 64; W > 64; W = 1
GRIDS = [(256, 32, 2, 2), (100, 24, 2, 2), (64, 80, 1, 1), (7, 1, 2, 2)]


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("TL,W,B,H", GRIDS)
def test_axial_kernels_against_float64(ops, TL, W, B, H, axis, dh):
    S = TL + W * W
    qkv, dout = _qkv(B, S, H, dh, _gen(TL * 7 + W + axis + dh))
    out, lse, dqkv = run_axial(ops, qkv, dout, (TL, W, axis))
    assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all()
    for n, v in ratios(qkv, dout, out, lse, dqkv, visible(S, TL, W, axis)).items():
        float64_bounds.report(f"{NAMES[axis]} TL={TL} W={W} dh={dh} {n}", v, TAG)


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("TL,W,B,H", GRIDS)
def test_segment_edges_are_exact(ops, TL, W, B, H, axis):
    """q = 0: lse_i = log(#keys query i sees).  The kernel passes against the oracle and fails against the oracle
    whose segments are shifted by one key (the previous row's last token / the neighbouring column)."""
    S, dh = TL + W * W, 64
    qkv, dout = _qkv(B, S, H, dh, _gen(TL + 3 * W + axis))
    qkv[:, :, 0] = 0
    out, lse, dqkv = run_axial(ops, qkv, dout, (TL, W, axis))
    mask = visible(S, TL, W, axis)
    assert max(ratios(qkv, dout, out, lse, dqkv, mask).values()) < 1.0
    assert (lse.to(F64) - torch.log(mask.sum(-1).to(F64))).abs().max() < 1e-5
    if W > 1:
        for shift in (-1, 1):
            got = max(ratios(qkv, dout, out, lse, dqkv, visible(S, TL, W, axis, shift)).values())
            print(f"[{TAG}] {NAMES[axis]} TL={TL} W={W} against the segment shifted by {shift}: worst {got:.1f}")
            assert got > 1.0, shift


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("axis", [0, 1])
def test_dominating_key_outside_the_segment_is_not_seen(ops, axis, dh):
    """Every image query's key just outside its segment (the previous row's last token for row layers, the left
    neighbour in the same row for column layers) gets a huge logit: the kernel output must not follow it."""
    TL, W, B, H = 100, 24, 1, 2
    S = TL + W * W
    qkv, dout = _qkv(B, S, H, dh, _gen(5 + axis + dh))
    q = torch.zeros(B, S, H, dh, device=DEV)
    q[..., 0] = 1.0
    k = torch.zeros(B, S, H, dh, device=DEV)
    k[..., 0] = 0.01 * torch.randn(B, S, H, device=DEV, generator=_gen(1))
    # keys whose row (axis 0) ends / column (axis 1) index is W - 1: the neighbour one key back of the next segment
    kk = torch.arange(S, device=DEV) - TL
    edge = (kk >= 0) & ((kk % W == W - 1) if axis == 0 else (kk % W == W - 2))
    k[:, edge, :, 0] = 8.0
    qkv[:, :, 0], qkv[:, :, 1] = q.to(BF16), k.to(BF16)
    out, lse, dqkv = run_axial(ops, qkv, dout, (TL, W, axis))
    res = ratios(qkv, dout, out, lse, dqkv, visible(S, TL, W, axis))
    assert max(res.values()) < 1.0, res
    wrong = max(ratios(qkv, dout, out, lse, dqkv, visible(S, TL, W, axis, 1)).values())
    print(f"[{TAG}] {NAMES[axis]} dh={dh} dominating key against the shifted segment: worst {wrong:.1f}")
    assert wrong > 1.0


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("TL,W", [(256, 32), (100, 24), (64, 80)])
def test_prefill_lengths(ops, TL, W, axis):
    """A prompt prefill runs the kernels at S = P < TL + W^2: absent rows are neither seen nor stored."""
    N, B, H, dh = TL + W * W, 1, 2, 128
    qkv_full, dout_full = _qkv(B, N, H, dh, _gen(TL + W + axis))
    for P in (TL, TL + 1, TL + W - 1, TL + W + 5, N - 1):
        qkv, dout = qkv_full[:, :P].contiguous(), dout_full[:, :P].contiguous()
        out, lse, dqkv = run_axial(ops, qkv, dout, (TL, W, axis))
        for n, v in ratios(qkv, dout, out, lse, dqkv, visible(P, TL, W, axis)).items():
            float64_bounds.report(f"prefill {NAMES[axis]} TL={TL} W={W} P={P} {n}", v, TAG)


def test_invalid_axial_geometry_is_rejected(ops):
    from dalle_mtf_b200 import lib as L
    lib = L.load()
    B, S, H, dh = 1, 20, 1, 64
    qkv = torch.zeros(B, S, 3, H, dh, dtype=BF16, device=DEV)
    out, lse = torch.zeros(B, S, H, dh, dtype=BF16, device=DEV), torch.zeros(B, H, S, device=DEV)
    kc = torch.zeros(B, S, H, dh, dtype=BF16, device=DEV)
    step = torch.zeros(B, 3, H, dh, dtype=BF16, device=DEV)
    pos = torch.zeros(1, dtype=I32, device=DEV)
    s = L.stream_ptr()
    for TL, W, axis in ((4, 4, 2), (4, 4, -1), (4, 0, 0), (-1, 5, 0), (3, 4, 1)):   # last: S = 20 > 3 + 16
        assert lib.db200_attn_axial_fwd(s, qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, S, H, dh, TL, W, axis,
                                        1.0) != 0
        assert lib.db200_attn_axial_bwd(s, qkv.data_ptr(), out.data_ptr(), out.data_ptr(), lse.data_ptr(), None,
                                        lse.data_ptr(), qkv.data_ptr(), B, S, H, dh, TL, W, axis, 1.0) != 0
        assert lib.db200_attn_decode_axial(s, step.data_ptr(), kc.data_ptr(), kc.data_ptr(), out.data_ptr(), B, S, H,
                                           dh, 3, TL, W, axis, 1.0) != 0
        assert lib.db200_attn_decode_axial_dev(s, step.data_ptr(), kc.data_ptr(), kc.data_ptr(), out.data_ptr(), B, S,
                                               H, dh, pos.data_ptr(), TL, W, axis, 1.0) != 0
    with pytest.raises(L.DB200Error):
        ops.attn_fwd(qkv, out, lse, B, S, H, dh, 1.0, radius=4, axial=(4, 4, 0))
    with pytest.raises(L.DB200Error):
        ops.attn_fwd(qkv, out, lse, B, S, H, dh, 1.0, axial=(4, 4, 0), dropout=L.make_dropout(0.1, 0, 0, 2, 0))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- decode
@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("axis", [0, 1])
def test_attn_decode_axial_against_float64(ops, axis, dh):
    TL, W = 256, 32
    B, S, H = 4, TL + W * W, 512 // dh
    g = _gen(dh + axis)
    vis = visible(S, TL, W, axis)
    positions = (0, 100, TL - 1, TL, TL + 1, TL + W - 1, TL + W, TL + 5 * W, TL + 6 * W - 1, TL + 17 * W + 9, S - W,
                 S - 1)
    for pos in positions:
        kc = (torch.randn(B, S, H, dh, generator=g, device=DEV) * 1.3 * dh ** -0.25).to(BF16)
        vc = torch.randn(B, S, H, dh, generator=g, device=DEV).to(BF16)
        step = torch.randn(B, 3, H, dh, generator=g, device=DEV)
        step[:, :2] *= 1.3 * dh ** -0.25
        step = step.to(BF16)
        kc2, vc2 = kc.clone(), vc.clone()
        out = nan_like((B, H, dh), BF16)
        ops.attn_decode(step, kc, vc, out, pos, 1.0, axial=(TL, W, axis))
        assert torch.equal(kc[:, pos], step[:, 1]) and torch.equal(vc[:, pos], step[:, 2])
        keys = vis[pos].nonzero()[:, 0]
        ref, absref, b = decode_reference(step[:, 0], kc[:, keys], vc[:, keys], 1.0)
        float64_bounds.check(f"attn_decode {NAMES[axis]} dh={dh} pos={pos}", out, ref, absref, b=b, bf16_out=True,
                             tag=TAG)
        pos_dev = torch.full((1,), pos, dtype=I32, device=DEV)
        out_dev = nan_like((B, H, dh), BF16)
        ops.attn_decode_dev(step, kc2, vc2, out_dev, pos_dev, 1.0, axial=(TL, W, axis))
        assert torch.equal(out_dev, out) and torch.equal(kc2, kc) and torch.equal(vc2, vc)


# ------------------------------------------------------------------------------------------------------- engine
# d, layers, H, text vocab, image vocab, text len, image len (W^2), B, layer types
CASES = [(256, 3, 2, 1000, 100, 40, 25, 3, ("axial_row", "axial_col", "global")),
         (256, 3, 4, 1000, 100, 100, 64, 2, ("global", "axial_col", "local")),
         (512, 2, 4, 3000, 512, 70, 100, 2, ("axial_col", "axial_row"))]


def _case(d, Ly, H, tv, iv, ts, isl, B, types, recompute=False, rates=(0.0, 0.0, 0.0), dseed=0, seed=0):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    cfg = OA.AxialConfig(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=48)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if k.endswith("/g"):
            params[k] = 1 + torch.randn(params[k].shape, generator=g) * 0.05
    tokens = torch.randint(0, cfg.total_tokens - 1, (B, cfg.seq_len), generator=g)
    eng = DalleEngine(d, Ly, H, tv, iv, ts, isl, recompute_grad=recompute, dropout=rates, dropout_seed=dseed,
                      attention_types=types, local_attention_radius=48)
    eng.load_params(params)
    return cfg, params, tokens, eng


@pytest.mark.parametrize("rates", [(0.0, 0.0, 0.0), RATES], ids=["no-dropout", "dropout"])
@pytest.mark.parametrize("case", CASES)
def test_mixed_engine_matches_the_oracle_recompute_off_and_on(case, rates):
    step, row0, dseed = 6, 1, 11
    spec = (rates, dseed, step, row0)
    cfg, params, tokens, _ = _case(*case, rates=rates, dseed=dseed)
    loss32, _, logits32, g32 = OA.loss_and_grads(params, tokens, cfg, spec, bf16=False)
    _, _, logits16, g16 = OA.loss_and_grads(params, tokens, cfg, spec, bf16=True)
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
    # the axial layers matter: the same weights as an all-global model give another loss
    gcfg = OA.AxialConfig(*case[:7])
    assert abs(OA.loss_and_grads(params, tokens, gcfg, spec)[0].item() - loss32.item()) > 1e-4


def _three_steps(types, rates=RATES):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    eng = DalleEngine(256, 3, 2, 500, 64, 60, 64, dropout=rates, dropout_seed=1, attention_types=types)
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


def test_axial_training_is_bitwise_reproducible_and_calls_the_axial_kernels(monkeypatch):
    from dalle_mtf_b200 import lib as L, ops
    from dalle_mtf_b200.dalle_engine import DalleEngine
    lib = L.load()
    seen = []
    for name in ("db200_attn_causal_fwd", "db200_attn_causal_fwd_ex", "db200_attn_causal_bwd",
                 "db200_attn_causal_bwd_ex", "db200_attn_local_fwd", "db200_attn_local_bwd", "db200_attn_axial_fwd",
                 "db200_attn_axial_bwd"):
        fn = getattr(lib, name)
        # axial calls are recorded with their (text_len, grid_w, axis)
        monkeypatch.setattr(lib, name, lambda *a, _fn=fn, _n=name: (
            seen.append((_n,) + (tuple(a[-4:-1]) if "axial" in _n else ())), _fn(*a))[1])
    types = ["axial_row", "global", "axial_col"]
    a, pa = _three_steps(types)
    calls = list(seen)
    seen.clear()
    b, pb = _three_steps(types)
    for (la, ga), (lb, gb) in zip(a, b):
        assert torch.isfinite(ga).all() and torch.equal(la, lb) and torch.equal(ga, gb)
    assert torch.equal(pa, pb) and seen == calls
    # every step: the row layer, the global layer (with attention dropout), the column layer; backward reversed
    one_step = [("db200_attn_axial_fwd", 60, 8, 0), ("db200_attn_causal_fwd_ex",), ("db200_attn_axial_fwd", 60, 8, 1),
                ("db200_attn_axial_bwd", 60, 8, 1), ("db200_attn_causal_bwd_ex",), ("db200_attn_axial_bwd", 60, 8, 0)]
    assert calls == one_step * 3
    assert not torch.equal(_three_steps(["global"] * 3)[1], pa)
    eng = DalleEngine(256, 3, 2, 500, 64, 60, 64, dropout=RATES, dropout_seed=1, attention_types=types)
    dd = eng._dropout_descs(2, 0)
    assert dd["attn"][0] is None and dd["attn"][1] is not None and dd["attn"][2] is None
    assert ops.attn_pairs_axial(eng.S, 60, 8, 0) < ops.attn_pairs(eng.S)


# ------------------------------------------------------------------------------------------------------- generation
GEN = [(256, 3, 2, 300, 64, 24, 36, 3, ("axial_row", "axial_col", "global"), 29),
       (256, 3, 4, 500, 100, 70, 81, 2, ("axial_col", "local", "axial_row"), 77)]


def _sharp(d, Ly, H, tv, iv, ts, isl, types):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    cfg = OA.AxialConfig(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=20)
    params = O.init_params(cfg, 3)
    g = torch.Generator().manual_seed(9)
    for k in params:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if "wte" in k or "wout" in k or k.endswith("kernel"):
            params[k] = params[k] * 4
    eng = DalleEngine(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=20)
    eng.load_params(params)
    return eng, params, cfg


@pytest.mark.parametrize("d,Ly,H,tv,iv,ts,isl,B,types,P", GEN)
def test_axial_generation_follows_the_full_forward_pass(d, Ly, H, tv, iv, ts, isl, B, types, P):
    from dalle_mtf_b200.sampling import DalleSampler
    eng, params, cfg = _sharp(d, Ly, H, tv, iv, ts, isl, types)
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
    _, _, logits32, _ = OA.loss_and_grads(params, toks.cpu().long(), cfg, bf16=False)
    assert relfro(dec, logits32[:, :S - 1]) < 3e-2
    assert torch.equal(smp.generate_graphed(text, temperature=0.0), toks)
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
    out = smp.complete(text, toks[:, ts:P] - tv, temperature=0)
    assert torch.equal(out[:, :P], toks[:, :P]) and (out[:, P:] >= tv).all() and (out[:, P:] < tv + iv).all()


def test_guided_generation_runs_on_an_axial_model():
    from dalle_mtf_b200.sampling import DalleSampler
    eng, _, _ = _sharp(256, 3, 2, 300, 64, 24, 36, ("axial_row", "axial_col", "global"))
    smp = DalleSampler(eng)
    text = torch.randint(0, 299, (3, 24), generator=torch.Generator().manual_seed(2)).to(I32).cuda()
    eager = smp.generate(text, temperature=0.0, guidance_scale=3.0)
    graphed = smp.generate_graphed(text, temperature=0.0, guidance_scale=3.0)
    assert torch.equal(eager, graphed) and torch.equal(eager[:, :24], text)
    assert ((eager[:, 24:] >= 300) & (eager[:, 24:] < 364)).all()
    torch.manual_seed(0)
    a = smp.complete(text, samples_per_prompt=2, temperature=1.0, guidance_scale=3.0, top_k=8)
    torch.manual_seed(0)
    b = smp.complete(text, samples_per_prompt=2, temperature=1.0, guidance_scale=3.0, top_k=8)
    assert torch.equal(a, b) and a.shape == (6, 60) and ((a[:, 24:] >= 300) & (a[:, 24:] < 364)).all()


def test_model_fn_trains_and_evaluates_with_axial_layers(tmp_path):
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
    axial = dict(attention_types=[[["axial_row", "axial_col"], 1]])
    spec = dalle_model_fn(img, cap, "train", params(**axial))
    W = math.isqrt(spec.engine.image_seq_len)
    assert spec.engine.axial == [(12, W, 0), (12, W, 1)]
    losses = [spec.train_op(img, cap).item() * spec.loss_scale for _ in range(2)]
    ev = spec.eval_op(img, cap).item() * spec.loss_scale
    assert all(math.isfinite(x) and 0 < x < 20 for x in losses + [ev])
    plain = dalle_model_fn(img, cap, "eval", params())
    ev_axial = dalle_model_fn(img, cap, "eval", params(**axial)).eval_op(img, cap).item()
    assert ev_axial != plain.eval_op(img, cap).item()
