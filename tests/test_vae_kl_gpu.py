"""GPU tests of the discrete VAE's KL term: the kernels against float64, the engine and the model boundary against the
oracle (oracle/vae_kl.py).

Kernels (db200_vae_kl_stats, db200_gumbel_softmax_bwd_kl), checked per element against float64 on the same fp32 inputs.
eps = 2^-24; n = K / 32 + 40 bounds the sequential fp32 operations one lane's running sums and the five shuffle merges
take per row (each contributes at most eps relative; expf / logf add <= 2 ulp each, folded into the +40).  With
A_r = sum_k q_rk |l_rk - lse_r| (float64) and M_r = max_k |l_rk|:
  * lse_r:  s = sum exp(l - m) is within n eps relative, so log s within n eps absolute, and m + log s adds one rounding:
            |d lse| <= n eps + 4 eps (|lse| + M).
  * e_r = t / s - log s and KL_r = t / s - log(s / K): t = sum exp(l - m)(l - m) carries n eps relative on
            sum q |l - m| <= A + 2 log K (l - m = (l - lse) + log s, log s <= log K), and every l - m is rounded once
            (eps M):  |d e|, |d KL_r| <= n eps (A + 2 log K + 2) + 8 eps M.  For near-uniform rows (std 1e-3) KL_r is
            ~5e-7 and the bound ~n eps (2 log K + 2) is an absolute one (cancellation case).
  * the KL sum: scale * sum_r KL_r, accumulated per warp in row order, then over the CTA's 8 warps, then in CTA order:
            |d sum| <= scale (sum_r bound_r + (rows + 64) eps sum_r |KL_r|) + eps |base + sum|.
  * backward, fed lse / e rounded from float64 (so it is tested on its own): z = l - lse carries
            dz <= eps (|lse| + |z|); exp(z) (dz + 2 eps) relative; (z - e) dz + eps (|e| + |z - e|); so the KL part
            c q (z - e) is within c q ((dz + 4 eps)(|z - e| + 1) + eps |e|) + c 2^-120 (|z - e| + 1) (the last term covers
            q that is subnormal in fp32); the straight-through part y (dy - dot) / tau within
            (n eps sum |y dy| + 3 eps (|dy| + |dot|)) y / tau.
  * code histogram: bit-exact against bincount of the first-maximum codes (ties to the first, NaN rows to code 0).
Outputs are NaN-filled first; accumulated outputs (KL sum, histogram) start from a non-zero base.

Engine and boundary: the fp32 step at the geometries of tests/test_engine_gpu.py's fp32 oracle test, the bf16 step
against the oracle's bf16 policy and the vae_coco geometry, with the same tolerances as those tests; mutated oracles must
fail them.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24


def relfro(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def ref_stats(logits):
    """float64 lse, e, KL_r and the per-row bounds of the module docstring for fp32 logits [rows, K] (any device)."""
    l = logits.double()
    K = l.shape[-1]
    lse = torch.logsumexp(l, -1)
    z = l - lse[:, None]
    q = z.exp()
    qz = torch.where(q > 0, q * z, torch.zeros_like(q))     # a -inf logit: q = 0 contributes 0
    e = qz.sum(-1)
    A = qz.abs().sum(-1)
    M = torch.where(torch.isinf(l), torch.zeros_like(l), l.abs()).amax(-1)
    n = K / 32 + 40
    b_e = n * EPS * (A + 2 * math.log(K) + 2) + 8 * EPS * M
    b_lse = n * EPS + 4 * EPS * (lse.abs() + M)
    return lse, e, e + math.log(K), b_lse, b_e


def run_stats(logits, base_kl=0.75, base_hist=3, guard=16):
    from dalle_mtf_b200 import ops
    rows, K = logits.shape
    lse = torch.full((rows + guard,), float("nan"), device=DEV)
    ent = torch.full((rows + guard,), float("nan"), device=DEV)
    hist = torch.full((K + guard,), base_hist, dtype=torch.int32, device=DEV)
    acc = torch.full((1,), base_kl, device=DEV)
    ops.vae_kl_stats(logits, lse, ent, hist, acc, rows, K, 1.0 / rows)
    torch.cuda.synchronize()
    assert torch.isnan(lse[rows:]).all() and torch.isnan(ent[rows:]).all()     # nothing past the last row
    assert (hist[K:] == base_hist).all()                                        # nothing past the last code
    return lse[:rows], ent[:rows], (hist[:K] - base_hist), acc - base_kl, acc


def check_stats(logits, finite_rows=None):
    from oracle import vae_kl as OK
    rows, K = logits.shape
    lse, ent, hist, kl, acc = run_stats(logits)
    ref_codes = torch.bincount(OK.first_max_codes(logits.cpu()), minlength=K)
    assert torch.equal(hist.cpu().long(), ref_codes)
    lse64, e64, kl64, b_lse, b_e = ref_stats(logits)
    sel = torch.ones(rows, dtype=torch.bool, device=DEV) if finite_rows is None else finite_rows.to(DEV)
    assert ((lse.double() - lse64).abs() <= b_lse)[sel].all()
    assert ((ent.double() - e64).abs() <= b_e)[sel].all()
    if finite_rows is None:
        total = kl64.sum() / rows
        bound = (b_e.sum() + (rows + 64) * EPS * kl64.abs().sum()) / rows + EPS * (0.75 + total.abs()) + EPS
        assert abs(kl.double().item() - total.item()) <= bound.item() + EPS * 2   # + the subtraction of the base
    return lse, ent, hist, kl


@pytest.mark.parametrize("rows,K", [(16384, 8192), (32768, 512), (37, 1), (1001, 7), (515, 100), (333, 8191),
                                    (130, 16384)])
def test_kl_stats_against_float64(rows, K):
    """Production shapes (vae_coco at 16 images per GPU, vae_example_b200), small and odd K, rows that leave the last
    CTA part-empty, and a K above the shared-memory histogram limit (global atomics)."""
    g = torch.Generator(device=DEV).manual_seed(rows + K)
    logits = torch.randn(rows, K, generator=g, device=DEV) * 2
    logits[:, :3] += 1.5   # some peaky rows, with ties of the maximum below
    logits[rows // 2, : min(K, 4)] = 9.0
    check_stats(logits)


@pytest.mark.parametrize("std", [1e-3, 30.0])
def test_kl_stats_near_uniform_and_dominating(std):
    """std 1e-3: KL_r ~ 5e-7, cancellation case (absolute bound).  std 30: q underflows to 0 on most codes, no NaN."""
    g = torch.Generator(device=DEV).manual_seed(5)
    logits = torch.randn(4099, 8192, generator=g, device=DEV) * std
    lse, ent, hist, kl = check_stats(logits)
    assert torch.isfinite(lse).all() and torch.isfinite(ent).all() and math.isfinite(kl.item())


def test_kl_stats_constant_rows_and_ties():
    logits = torch.zeros(64, 100, device=DEV)
    logits[1::2, 10] = 1.0
    logits[1::2, 20] = 1.0         # tie: the first maximum, code 10
    lse, ent, hist, kl = check_stats(logits)
    assert hist[0].item() == 32 and hist[10].item() == 32


def test_kl_stats_non_finite_rows_stay_in_their_row():
    g = torch.Generator(device=DEV).manual_seed(6)
    rows, K = 200, 300
    logits = torch.randn(rows, K, generator=g, device=DEV)
    bad = torch.zeros(rows, dtype=torch.bool)
    for r, col, v in ((3, 5, float("nan")), (4, 0, float("inf")), (50, 299, float("-inf")), (51, 7, float("nan")),
                      (199, 150, float("inf"))):
        logits[r, col] = v
        bad[r] = True
    logits[120, :] = float("-inf")
    bad[120] = True
    logits[121, 17] = float("-inf")            # one -inf code in a finite row: q = 0 there, the row stays exact
    lse, ent, hist, _ = check_stats(logits, finite_rows=~bad)
    assert hist.sum().item() == rows
    assert torch.isfinite(lse[121]) and torch.isfinite(ent[121])


def test_kl_stats_and_backward_are_bit_reproducible():
    from dalle_mtf_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(7)
    rows, K = 16384, 8192
    logits = torch.randn(rows, K, generator=g, device=DEV) * 3
    y = torch.softmax(torch.randn(rows, K, generator=g, device=DEV), -1)
    dy = torch.randn(rows, K, generator=g, device=DEV)
    outs = []
    for _ in range(2):
        lse, ent, hist, kl, _ = run_stats(logits)
        dl = torch.full((rows, K), float("nan"), device=DEV)
        ops.gumbel_softmax_bwd_kl(y, dy, logits, lse, ent, dl, rows, K, 0.8, 0.3 / rows)
        torch.cuda.synchronize()
        outs.append((kl.clone(), hist.clone(), dl))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert torch.equal(outs[0][2], outs[1][2])


def check_backward(logits, y, dy, tau, c, rows_sel=None):
    """dlogits of gumbel_softmax_bwd_kl (fed float64 lse / e rounded to fp32) against float64 with the docstring bound;
    returns dlogits.  rows_sel: check only these rows (large cases)."""
    from dalle_mtf_b200 import ops
    rows, K = logits.shape
    lse64, e64, _, _, _ = ref_stats(logits) if rows_sel is None else (None,) * 5
    if rows_sel is not None:
        l_sel = logits[rows_sel]
        ls, es, _, _, _ = ref_stats(l_sel)
        lse32 = torch.zeros(rows, device=DEV)
        ent32 = torch.zeros(rows, device=DEV)
        lse32[rows_sel], ent32[rows_sel] = ls.float(), es.float()
    else:
        lse32, ent32 = lse64.float(), e64.float()
    dl = torch.full((rows, K), float("nan"), device=DEV)
    ops.gumbel_softmax_bwd_kl(y, dy, logits, lse32, ent32, dl, rows, K, tau, c)
    torch.cuda.synchronize()
    idx = torch.arange(rows, device=DEV) if rows_sel is None else rows_sel
    l, yy, d, got = logits[idx].double(), y[idx].double(), dy[idx].double(), dl[idx].double()
    ls, es = lse32[idx].double(), ent32[idx].double()
    z = l - ls[:, None]
    q = z.exp()
    dot = (yy * d).sum(-1, keepdim=True)
    ref = yy * (d - dot) / tau + c * q * (z - es[:, None])
    n = K / 32 + 40
    dz = EPS * (ls.abs()[:, None] + z.abs())
    zc = (z - es[:, None]).abs()
    b_kl = c * q * ((dz + 4 * EPS) * (zc + 1) + EPS * es.abs()[:, None]) + c * 2.0 ** -120 * (zc + 1)
    b_st = (n * EPS * (yy * d).abs().sum(-1, keepdim=True) + 3 * EPS * (d.abs() + dot.abs())) * yy / tau
    err = (got - ref).abs()
    assert (err <= b_kl + b_st + 1e-37).all(), (err - b_kl - b_st).max().item()
    return dl


@pytest.mark.parametrize("rows,K,std", [(16384, 8192, 2.0), (32768, 512, 2.0), (37, 1, 1.0), (1001, 7, 1.0),
                                        (515, 100, 1.0), (333, 8191, 1.0), (2049, 8192, 1e-3), (2049, 8192, 30.0)])
def test_kl_backward_against_float64(rows, K, std):
    g = torch.Generator(device=DEV).manual_seed(rows * 3 + K)
    logits = torch.randn(rows, K, generator=g, device=DEV) * std
    y = torch.softmax(torch.randn(rows, K, generator=g, device=DEV) * 2, -1)
    dy = torch.randn(rows, K, generator=g, device=DEV) * 1e-3
    dl = check_backward(logits, y, dy, 0.7, 5.0 / rows)
    assert torch.isfinite(dl).all()


def test_kl_backward_with_zero_weight_is_the_plain_backward():
    from dalle_mtf_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(8)
    rows, K = 1000, 512
    logits = torch.randn(rows, K, generator=g, device=DEV)
    y = torch.softmax(torch.randn(rows, K, generator=g, device=DEV), -1)
    dy = torch.randn(rows, K, generator=g, device=DEV)
    lse, ent, _, _, _ = run_stats(logits)
    a = torch.full((rows, K), float("nan"), device=DEV)
    b = torch.full((rows, K), float("nan"), device=DEV)
    ops.gumbel_softmax_bwd(y, dy, a, rows, K, 0.9)
    ops.gumbel_softmax_bwd_kl(y, dy, logits, lse, ent, b, rows, K, 0.9, 0.0)
    assert torch.equal(a, b)


def test_kl_kernels_past_2_31_elements():
    """rows * K >= 2^31 (64-bit row offsets): sampled rows per element, the KL sum and the histogram's total."""
    K = 8192
    rows = (1 << 31) // K + 5
    g = torch.Generator(device=DEV).manual_seed(9)
    logits = torch.randn(rows, K, generator=g, device=DEV) * 2
    lse, ent, hist, kl, _ = run_stats(logits)
    assert hist.sum().item() == rows
    sel = torch.cat([torch.arange(0, 8), torch.randint(0, rows, (48,), generator=torch.Generator().manual_seed(0)),
                     torch.arange(rows - 8, rows)]).to(DEV)
    lse64, e64, kl64, b_lse, b_e = ref_stats(logits[sel])
    assert ((lse[sel].double() - lse64).abs() <= b_lse).all() and ((ent[sel].double() - e64).abs() <= b_e).all()
    total, bsum, asum = 0.0, 0.0, 0.0
    for r0 in range(0, rows, 8192):          # float64 sum in slabs
        _, _, k64, _, be = ref_stats(logits[r0:r0 + 8192])
        total += k64.sum().item(); bsum += be.sum().item(); asum += k64.abs().sum().item()
    bound = (bsum + (rows + 64) * EPS * asum) / rows + EPS * (0.75 + abs(total / rows)) + 2 * EPS
    assert abs(kl.item() - total / rows) <= bound
    del lse, ent
    y = torch.empty_like(logits).fill_(1.0 / K)
    dy = torch.randn(rows, K, generator=g, device=DEV) * 1e-3
    check_backward(logits, y, dy, 1.0, 2.0 / rows, rows_sel=sel)


def test_kl_entry_points_reject_bad_arguments():
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops
    x = torch.zeros(8, 4, device=DEV)
    r = torch.zeros(8, device=DEV)
    h = torch.zeros(4, dtype=torch.int32, device=DEV)
    with pytest.raises(L.DB200Error):
        ops.vae_kl_stats(x, r, r, h, r[:1], 8, 4, float("nan"))
    with pytest.raises(L.DB200Error):
        ops.gumbel_softmax_bwd_kl(x, x, x, r, r, x, 8, 4, 1.0, float("inf"))
    with pytest.raises(L.DB200Error):
        ops.gumbel_softmax_bwd_kl(x, x, x, r, r, x, 0, 4, 1.0, 1.0)
    s = L.stream_ptr()
    assert L.load().db200_vae_kl_stats(s, x.data_ptr(), r.data_ptr(), r.data_ptr(), h.data_ptr(), r.data_ptr(), 8, 4,
                                       1.0, None, 0) != 0       # workspace missing
    assert L.load().db200_vae_kl_stats_workspace_bytes(8, 4) > 0


# ---------------------------------------------------------------------------------------------------------- engine
def _case(convblocks, K, size, B, seed, cb_scale=8.0):
    from oracle import vae as OV
    g = torch.Generator().manual_seed(seed)
    p = OV.init_params(convblocks, K, seed=seed)
    for k in p:
        if k.endswith("/bias"):
            p[k] = torch.randn(p[k].shape, generator=g) * 0.05
    p["codebook/codebook"] = p["codebook/codebook"] * cb_scale   # peaky logits: the KL gradient is not negligible
    img = torch.rand(B, size, size, 3, generator=g) * 2 - 1
    hw = size // (2 ** len(convblocks))
    u = torch.rand(B * hw * hw, K, generator=g).clamp_(1e-9, 1.0)
    return p, img, u, hw


def _engine_step(p, img, u, K, size, convblocks, tau, hard, beta, use_bf16=False):
    from dalle_mtf_b200.vae_engine import VaeEngine
    eng = VaeEngine(K, size, convblocks, use_bf16=use_bf16, kl=True)
    eng.load_params(p)
    eng.zero_grads()
    acc = torch.zeros(2, device=DEV)
    eng.forward(img.to(DEV), u.to(DEV), tau, hard, loss_accum=acc[:1], kl_weight=beta, kl_accum=acc[1:])
    eng.backward()
    torch.cuda.synchronize()
    return eng, acc.cpu(), eng.export_params(eng.grads)


@pytest.mark.parametrize("convblocks,K,size,B,hard,tau", [
    ([[2, 32], [2, 64]], 64, 16, 4, True, 1.0), ([[2, 32], [2, 64]], 64, 16, 4, False, 0.5),
    ([[3, 64], [3, 128], [3, 256]], 512, 32, 8, True, 1.0)])
def test_vae_engine_fp32_kl_step_matches_oracle(convblocks, K, size, B, hard, tau):
    from oracle import vae_kl as OK
    p, img, u, hw = _case(convblocks, K, size, B, K + size)
    beta = 0.5
    uv = u.view(B, hw, hw, K)
    loss, mse, kl, out, logits, grads = OK.loss_and_grads(p, img, uv, convblocks, tau, hard, kl_weight=beta)
    eng, acc, eg = _engine_step(p, img, u, K, size, convblocks, tau, hard, beta)
    assert relfro(acc[:1], mse.reshape(1)) < 1e-4 and relfro(acc[1:], kl.reshape(1)) < 1e-4
    assert relfro(acc[:1] + beta * acc[1:], loss.reshape(1)) < 1e-4
    counts, _, _ = OK.codebook_usage(eng._b["logits"].cpu())
    assert torch.equal(eng.code_counts().cpu().long(), counts)
    for k in grads:
        assert relfro(eg[k], grads[k]) < 2e-2, k
    # each mutated oracle is told apart: by the KL value, or by the codebook and encoder gradients
    enc0 = "encoder/block_0/layer_0/conv_downsample/kernel"
    for m in OK.MUTATIONS:
        _, _, klm, _, _, gm = OK.loss_and_grads(p, img, uv, convblocks, tau, hard, kl_weight=beta, mutate=m)
        value_ok = relfro(acc[1:], klm.reshape(1)) < 1e-4
        grads_ok = relfro(eg["codebook/codebook"], gm["codebook/codebook"]) < 2e-2 and relfro(eg[enc0], gm[enc0]) < 2e-2
        assert not (value_ok and grads_ok), m
        if m != "no_centring":
            assert not value_ok, m
        assert not grads_ok, m


def test_vae_engine_bf16_kl_step_within_the_bf16_policy():
    from oracle import vae_kl as OK
    cb, K, size, B = [[2, 64], [2, 128]], 128, 32, 4
    p, img, u, hw = _case(cb, K, size, B, 77)
    beta = 0.5
    uv = u.view(B, hw, hw, K)
    loss, mse, kl, _, _, grads = OK.loss_and_grads(p, img, uv, cb, 1.0, False, kl_weight=beta)
    _, _, kl16, _, _, g16 = OK.loss_and_grads(p, img, uv, cb, 1.0, False, bf16=True, kl_weight=beta)
    eng, acc, eg = _engine_step(p, img, u, K, size, cb, 1.0, False, beta, use_bf16=True)
    assert relfro(acc[:1] + beta * acc[1:], loss.reshape(1)) < 2e-2
    assert relfro(acc[1:], kl.reshape(1)) <= 1.5 * relfro(kl16.reshape(1), kl.reshape(1)) + 2e-2
    for k in grads:
        e_engine, e_ref = relfro(eg[k], grads[k]), relfro(g16[k], grads[k])
        assert e_engine <= 1.5 * e_ref + 2e-2, (k, e_engine, e_ref)


def test_vae_coco_geometry_k8192_bf16_kl_step():
    """configs/vae_coco_b200.json geometry: 256 px, [[2,128],[3,256],[5,512]], K = 8192, bf16, soft Gumbel, B = 1."""
    import os
    from oracle import vae_kl as OK
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    cb, K, size, B, tau = [[2, 128], [3, 256], [5, 512]], 8192, 256, 1, 0.7
    p, img, u, hw = _case(cb, K, size, B, 21, cb_scale=4.0)
    beta = 1.0
    uv = u.view(B, hw, hw, K)
    loss, mse, kl, _, _, grads = OK.loss_and_grads(p, img, uv, cb, tau, False, kl_weight=beta)
    _, _, kl16, _, _, g16 = OK.loss_and_grads(p, img, uv, cb, tau, False, bf16=True, kl_weight=beta)
    eng, acc, eg = _engine_step(p, img, u, K, size, cb, tau, False, beta, use_bf16=True)
    assert relfro(acc[:1] + beta * acc[1:], loss.reshape(1)) < 2e-2
    assert relfro(acc[1:], kl.reshape(1)) <= 1.5 * relfro(kl16.reshape(1), kl.reshape(1)) + 2e-2
    for k in grads:
        e_engine, e_ref = relfro(eg[k], grads[k]), relfro(g16[k], grads[k])
        assert e_engine <= 1.5 * e_ref + 2e-2, (k, e_engine, e_ref)


def _record_ops(monkeypatch):
    """Wraps every function of dalle_mtf_b200.ops so that calls through the module are recorded by name."""
    import inspect
    from dalle_mtf_b200 import ops
    calls = []
    for name, fn in list(vars(ops).items()):
        if inspect.isfunction(fn) and fn.__module__ == ops.__name__ and not name.startswith("_"):
            def wrap(*a, _fn=fn, _name=name, **k):
                calls.append(_name)
                return _fn(*a, **k)
            monkeypatch.setattr(ops, name, wrap)
    return calls


@pytest.mark.parametrize("use_bf16", [False, True])
def test_launch_sequences_without_kl_and_with_zero_weight(monkeypatch, use_bf16):
    from dalle_mtf_b200.vae_engine import VaeEngine
    cb, K, size, B = [[2, 64], [2, 64]], 64, 16, 2
    p, img, u, _ = _case(cb, K, size, B, 3)
    seqs = {}
    for key, kl in (("absent", None), ("zero", 0.0), ("positive", 0.3)):
        eng = VaeEngine(K, size, cb, use_bf16=use_bf16, kl=kl is not None)
        eng.load_params(p)
        eng.zero_grads()
        calls = _record_ops(monkeypatch)
        eng.forward(img.to(DEV), u.to(DEV), 1.0, True, kl_weight=kl)
        eng.backward()
        eng.optimizer_step(1e-3, 1)
        torch.cuda.synchronize()
        seqs[key] = list(calls)
        monkeypatch.undo()
    new = {"vae_kl_stats", "gumbel_softmax_bwd_kl"}
    assert not new & set(seqs["absent"])
    assert [c for c in seqs["zero"] if c != "vae_kl_stats"] == seqs["absent"]
    assert seqs["zero"].count("vae_kl_stats") == 1
    assert [c if c != "gumbel_softmax_bwd_kl" else "gumbel_softmax_bwd" for c in seqs["positive"]] == seqs["zero"]


def test_kl_aux_slot_rides_the_first_bucket():
    from dalle_mtf_b200.vae_engine import VaeEngine
    cb, K, size, B = [[2, 64], [2, 64]], 64, 16, 2
    p, img, u, _ = _case(cb, K, size, B, 4)
    eng = VaeEngine(K, size, cb, kl=True)
    eng.load_params(p)
    eng.zero_grads()
    ranges = []
    eng.forward(img.to(DEV), u.to(DEV), 1.0, True, kl_weight=0.2)
    eng.backward(on_bucket_ready=lambda s, e: ranges.append((s, e)))
    s, e = ranges[0]
    assert s <= eng.aux_off < eng.aux_off + 1 < e
    torch.cuda.synchronize()
    assert eng.grads[eng.aux_off + 1].item() > 0


# -------------------------------------------------------------------------------------------------------- boundary
def _vae_params(tmp_path, **extra):
    from collections import defaultdict
    d = {"model_type": "vae", "num_tokens": 64, "convblocks": [[2, 64], [2, 64]], "dataset": {"image_size": 16},
         "train_batch_size": 4, "eval_batch_size": 4, "lr": 1e-3, "model_path": str(tmp_path / "vae"),
         "n_channels": 3, "train_gumbel_hard": True, "iterations": 2, "steps_per_checkpoint": 2, "train_steps": 6}
    d.update(extra)
    return defaultdict(lambda: None, d)


def test_vae_model_fn_anneal_matches_oracle_each_step(tmp_path):
    from dalle_mtf_b200.model_fns import TRAIN, EVAL, vae_model_fn
    from oracle import vae_kl as OK
    params = _vae_params(tmp_path, kl_loss_weight=0.8, kl_anneal_steps=2)
    g = torch.Generator().manual_seed(11)
    img = torch.rand(4, 16, 16, 3, generator=g) * 2 - 1
    u = torch.rand(4 * 16, 64, generator=g).clamp_(1e-9, 1.0)
    params["_gumbel_u"] = u.to(DEV)
    spec = vae_model_fn(img, img, TRAIN, params)
    cb = [[2, 64], [2, 64]]
    for step in range(4):
        p = spec.engine.export_params()
        beta_t = OK.kl_weight(step, params)
        loss, mse, kl, _, _, _ = OK.loss_and_grads(p, img, u.view(4, 4, 4, 64), cb, 1.0, True, kl_weight=beta_t)
        spec.train_op(img)
        assert spec.kl_weight == pytest.approx(beta_t)
        got = float(spec.loss_sum.item()) * spec.loss_scale
        parts = spec.loss_parts.cpu()
        assert abs(got - loss.item()) <= 1e-4 * abs(loss.item())
        assert relfro(parts[:1], mse.reshape(1)) < 1e-4 and relfro(parts[1:], kl.reshape(1)) < 1e-4
    used, ppl = spec.codebook_usage()
    counts, used_ref, ppl_ref = OK.codebook_usage(spec.engine._b["logits"].cpu())
    assert used == used_ref and ppl == pytest.approx(ppl_ref, rel=1e-12)
    # eval reports the same parts, at the training step's beta_t
    ev = vae_model_fn(img, img, EVAL, params)
    ev.engine.copy_params_from(spec.engine)
    ev.global_step = spec.global_step
    ev.eval_op(img)
    assert ev.loss_parts is not None and ev.loss_parts.numel() == 2 and ev.kl_weight == pytest.approx(0.8)
    got = float(ev.loss_sum.item()) * ev.loss_scale
    pe = ev.loss_parts.cpu()
    assert got == pytest.approx(pe[0].item() + 0.8 * pe[1].item(), rel=1e-6)


def test_vae_model_fn_resume_continues_the_schedule(tmp_path):
    from functools import partial
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.input_fns import vae_input_fn
    from dalle_mtf_b200.model_fns import vae_model_fn
    params = _vae_params(tmp_path, kl_loss_weight=1.0, kl_anneal_steps=8)
    est = Estimator(vae_model_fn, params)
    spec = est.train(partial(vae_input_fn, eval=False), max_steps=2)
    assert spec.kl_weight == pytest.approx(1 / 8)          # beta_t of the step run at global_step 1
    est.close()
    est2 = Estimator(vae_model_fn, params)
    spec2 = est2.train(partial(vae_input_fn, eval=False), max_steps=3)
    assert spec2.global_step == 3 and spec2.kl_weight == pytest.approx(2 / 8)
    est2.close()


def test_discrete_vae_model_returns_the_objective():
    from dalle_mtf_b200.models import DiscreteVAE
    from oracle import vae_kl as OK
    vae = DiscreteVAE(64, 16, [[2, 64], [2, 64]], kl_loss_weight=0.25)
    img = torch.rand(2, 16, 16, 3, generator=torch.Generator().manual_seed(0)) * 2 - 1
    loss, out = vae.forward(img, return_recon_loss=True)
    parts = vae.loss_parts.cpu()
    assert loss.item() == pytest.approx(parts[0].item() + 0.25 * parts[1].item(), rel=1e-6)
    ref_kl = OK.kl_uniform(vae.engine._b["logits"].double().cpu())
    assert parts[1].item() == pytest.approx(ref_kl.item(), rel=1e-5)
    plain = DiscreteVAE(64, 16, [[2, 64], [2, 64]])
    acc, _ = plain.forward(img, return_recon_loss=True)
    assert acc.numel() == 1 and plain.loss_parts is None
    with pytest.raises(ValueError):
        DiscreteVAE(64, 16, [[2, 64], [2, 64]], kl_loss_weight=-1.0)


def test_kl_trained_vae_checkpoint_feeds_dalle_model_fn(tmp_path):
    """The two-stage path of tests/test_engine_gpu.py with a KL-trained VAE: same checkpoint layout, tokens exact."""
    from collections import defaultdict
    from functools import partial
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.input_fns import dalle_input_fn, vae_input_fn
    from dalle_mtf_b200.model_fns import dalle_model_fn, vae_model_fn
    from dalle_mtf_b200.utils import latest_checkpoint, load_checkpoint
    from oracle import vae as OV
    vae_p = _vae_params(tmp_path, kl_loss_weight=0.1, steps_per_checkpoint=3)
    est = Estimator(vae_model_fn, vae_p)
    est.train(partial(vae_input_fn, eval=False), max_steps=6)
    est.close()
    st = load_checkpoint(latest_checkpoint(vae_p["model_path"]))
    vae_weights = {k[len("vae/"):]: v for k, v in st.items()
                   if k.startswith("vae/") and not k.endswith("/Adam") and not k.endswith("/Adam_1")}
    dalle_p = defaultdict(lambda: None, {"model_type": "dalle", "dataset": {"image_size": 16}, "train_batch_size": 4,
                                         "eval_batch_size": 4, "n_embd": 256, "n_layers": 2, "n_heads": 2,
                                         "text_vocab_size": 300, "image_vocab_size": 64, "text_seq_len": 12,
                                         "lr": 2e-3, "train_steps": 100, "warmup_steps": 2, "bf_16": True,
                                         "mesh_shape": "data:1", "layout": "batch_dim:data",
                                         "model_path": str(tmp_path / "dalle"), "iterations": 2,
                                         "steps_per_checkpoint": 4, "n_channels": 3, "padding_id": 299,
                                         "vae_params": vae_p})
    est2 = Estimator(dalle_model_fn, dalle_p)
    spec = est2.train(partial(dalle_input_fn, eval=False), max_steps=2)
    img, cap = next(iter(dalle_input_fn(dalle_p)))
    toks = spec.assemble(img, cap).cpu().long()
    assert torch.equal(toks[:, 12:], OV.encode_tokens(vae_weights, img, [[2, 64], [2, 64]]) + 300)
    est2.close()
