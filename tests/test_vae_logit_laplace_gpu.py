"""GPU tests of the discrete VAE's logit-Laplace reconstruction loss: the kernel against float64, the engine and the
model boundary against the oracle (oracle/vae_logit_laplace.py).

Kernel (db200_logit_laplace_fwd_bwd), per element against float64 on the same fp32 inputs.  eps = 2^-24; CUDA's
accurate expf / logf are within 2 ulp (<= 4 eps relative), and an IEEE division or fma rounds once.  For an input
x with |x| <= 1.5, mu, ln b (all fp32, exact in float64):
  * y = fma(0.4f, x, 0.5f) clamped to [0.1f, 0.9f]: 0.4f, 0.1f, 0.9f are within eps of 0.4, 0.1, 0.9, so
            |dy| <= 0.4 |x| eps + |y| eps + eps <= 3 eps.
  * ln y: |dy| / y + 4 eps |ln y| <= 30 eps + 10 eps;  1 - y rounds once (<= eps), so ln(1 - y) is within 40 eps + 10 eps;
            t = ln y - ln(1 - y) adds eps |t|:  |dt| <= 100 eps + eps |t|.
  * d = t - mu: |dd| <= |dt| + eps |d|;  1 / b = expf(-ln b): 4 eps relative;  a = |d| / b:
            |da| <= |dd| / b + 6 eps a.
  * nll = ln 2 + ln b + (ln y + ln(1 - y)) + a, ln 2 rounded (eps), four roundings on the running sum:
            |d nll| <= 100 eps + eps + |da| + 4 eps (1 + |ln b| + |ln y| + |ln(1 - y)| + a + |nll|).
  * d mu = -c sign(d) / b: within 6 eps c / b where |d| exceeds its error bound |dd|; elsewhere (d within rounding of 0)
            any of -c / b, 0, c / b is accepted.  t = mu exactly (x = 0 -> y = 0.5, t = 0; mu = 0) must give exactly 0.
  * d ln b = c (1 - a):  |err| <= c (|da| + 3 eps (1 + a)).
  * xhat = clamp(fma(2.5, 1 / (1 + expf(-mu)), -1.25), -1, 1): sigmoid within 7 eps relative, so |dxhat| <= 20 eps.
  * sums: each thread adds its V-channel items in order, then 5 shuffle levels, 8 warps, the scale, and the per-CTA
            partials in CTA order onto the base: k = V * items_per_thread + blocks + 20 sequential roundings at most, so
            |d sum| <= scale (sum_i bound_i + k eps sum_i |v_i|) + eps |base + sum|.
  * mse term (xhat - x)^2 with e = xhat - x: |err| <= 2 |e| (20 eps + eps |e|) + 2 eps e^2 + (20 eps)^2.
Outputs are NaN-filled with guard elements behind them; accumulated sums start from a non-zero base.

Engine and boundary: the fp32 step against the oracle at the tolerances of tests/test_vae_kl_gpu.py's fp32 KL step, the
bf16 step against the oracle's bf16 policy (vae_coco geometry included); mutated oracles must fail.
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


def near(a, b, tol=1e-4):
    """|a - b| <= tol max(|b|, 1) for scalars.  The mean NLL can sit near 0 (ln 2 + ln y + ln(1 - y) < 0 offsets
    |t - mu| / b), so its error is measured against the O(1) scale of the per-subpixel terms, not against itself."""
    a, b = float(a.reshape(-1)[0]), float(b.reshape(-1)[0])
    return abs(a - b) <= tol * max(abs(b), 1.0)


# ---------------------------------------------------------------------------------------------------------- kernel
def make_inputs(n_pix, Cp, seed):
    """stats [n_pix, 2 Cp] with ln b in [-8, 4], targets x in [-1, 1] with exact +-1 and out-of-range values, and
    t = mu exactly (x = 0, mu = 0) on a slice of pixels."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    mu = torch.randn(n_pix, Cp, generator=g, device=DEV) * 2
    lb = torch.rand(n_pix, Cp, generator=g, device=DEV) * 12 - 8
    x = torch.rand(n_pix, Cp, generator=g, device=DEV) * 2 - 1
    x[0::7] = 1.0
    x[3::7] = -1.0
    x[5::11] = torch.rand(x[5::11].shape, generator=g, device=DEV) * 3 - 1.5      # outside [-1, 1]: clamped
    x[1::13] = 0.0
    mu[1::13] = 0.0                                                              # t = mu exactly
    return torch.cat([mu, lb], -1).contiguous(), x.contiguous()


def ref64(stats, x):
    """float64 nll, d mu / c, d ln b / c, xhat, squared error and the per-element bounds of the module docstring."""
    Cp = x.shape[-1]
    s = stats.double()
    mu, lb, xd = s[:, :Cp], s[:, Cp:], x.double()
    y = (0.4 * xd + 0.5).clamp(0.1, 0.9)
    ly, l1y = torch.log(y), torch.log1p(-y)
    t = ly - l1y
    d = t - mu
    ib = torch.exp(-lb)
    a = d.abs() * ib
    nll = math.log(2) + lb + ly + l1y + a
    xh = (2.5 * torch.sigmoid(mu) - 1.25).clamp(-1, 1)
    e = xh - xd
    dt = 100 * EPS + EPS * t.abs()
    dd = dt + EPS * d.abs()
    da = dd * ib + 6 * EPS * a
    b_nll = 101 * EPS + da + 4 * EPS * (1 + lb.abs() + ly.abs() + l1y.abs() + a + nll.abs())
    b_se = 2 * e.abs() * (20 * EPS + EPS * e.abs()) + 2 * EPS * e * e + (20 * EPS) ** 2
    return dict(nll=nll, dmu=-torch.sign(d) * ib, dlb=1 - a, xh=xh, se=e * e, ib=ib, a=a, d=d, dd=dd, da=da,
                b_nll=b_nll, b_se=b_se)


def run_kernel(stats, x, scale, base=(0.75, -0.5), guard=16, decode=False):
    from dalle_mtf_b200 import ops
    n_pix, Cp = x.shape
    recon = torch.full((n_pix * Cp + guard,), float("nan"), device=DEV)
    if decode:
        ops.logit_laplace(stats, None, None, recon, None, None, n_pix, Cp, scale)
        torch.cuda.synchronize()
        assert torch.isnan(recon[n_pix * Cp:]).all()
        return recon[:n_pix * Cp].view(n_pix, Cp)
    dstats = torch.full((n_pix * 2 * Cp + guard,), float("nan"), device=DEV)
    nll = torch.full((1,), base[0], device=DEV)
    mse = torch.full((1,), base[1], device=DEV)
    ops.logit_laplace(stats, x, dstats, recon, nll, mse, n_pix, Cp, scale)
    torch.cuda.synchronize()
    assert torch.isnan(recon[n_pix * Cp:]).all() and torch.isnan(dstats[n_pix * 2 * Cp:]).all()
    return (recon[:n_pix * Cp].view(n_pix, Cp), dstats[:n_pix * 2 * Cp].view(n_pix, 2 * Cp), nll - base[0],
            mse - base[1], nll, mse)


def sum_terms(n_pix, Cp):
    """k of the module docstring for this launch."""
    from dalle_mtf_b200 import lib as L
    blocks = L.load().db200_logit_laplace_workspace_bytes(n_pix, Cp) // 8
    V = 4 if Cp % 4 == 0 else 1
    items = n_pix * (Cp // V)
    return V * -(-items // (blocks * 256)) + blocks + 20


def check_kernel(stats, x, scale=None):
    n_pix, Cp = x.shape
    c = 1.0 / (n_pix * Cp) if scale is None else scale
    xh, ds, nll, mse, nll_acc, mse_acc = run_kernel(stats, x, c)
    r = ref64(stats, x)
    assert ((xh.double() - r["xh"]).abs() <= 20 * EPS).all()
    assert (xh.abs() <= 1).all()
    # d mu
    dmu, dlb = ds[:, :Cp].double(), ds[:, Cp:].double()
    sure = r["d"].abs() > r["dd"]
    assert ((dmu - c * r["dmu"]).abs() <= 6 * EPS * c * r["ib"])[sure].all()
    assert (dmu.abs() <= c * r["ib"] * (1 + 6 * EPS))[~sure].all()
    exact = (x == 0) & (stats[:, :Cp] == 0)
    assert exact.any() and (ds[:, :Cp][exact] == 0).all()
    # d ln b
    assert ((dlb - c * r["dlb"]).abs() <= c * (r["da"] + 3 * EPS * (1 + r["a"]))).all()
    # the two sums
    k = sum_terms(n_pix, Cp)
    for got, acc, v, b, base in ((nll, nll_acc, r["nll"], r["b_nll"], 0.75), (mse, mse_acc, r["se"], r["b_se"], -0.5)):
        ref = c * v.sum().item()
        bound = c * (b.sum().item() + k * EPS * v.abs().sum().item()) + EPS * abs(base + ref) + 2 * EPS * abs(base)
        assert abs(got.double().item() - ref) <= bound, (got.item(), ref, bound)
    return xh, ds


@pytest.mark.parametrize("n_pix,Cp", [
    (16 * 256 * 256, 3),      # vae_coco_b200 per GPU (16 images)
    (32 * 256 * 256, 3),      # vae_example_b200 per GPU (32 images)
    (8 * 128 * 128, 12),      # stack_factor 2 (16-byte path)
    (1001, 12), (37, 3), (5, 1), (777, 7)])
def test_logit_laplace_kernel_against_float64(n_pix, Cp):
    stats, x = make_inputs(n_pix, Cp, n_pix + Cp)
    check_kernel(stats, x)


def test_logit_laplace_kernel_unaligned_rows_take_the_scalar_path():
    """Cp % 4 == 0 but the buffers start 4 bytes off a 16-byte boundary: the scalar instantiation, same results."""
    stats, x = make_inputs(513, 12, 3)
    s_off = torch.empty(stats.numel() + 1, device=DEV)[1:].view_as(stats)
    s_off.copy_(stats)
    x_off = torch.empty(x.numel() + 1, device=DEV)[1:].view_as(x)
    x_off.copy_(x)
    xh_a, ds_a = check_kernel(s_off, x_off, scale=0.01)
    xh_b, ds_b, *_ = run_kernel(stats, x, 0.01)
    assert torch.equal(xh_a, xh_b) and torch.equal(ds_a, ds_b)


@pytest.mark.parametrize("n_pix,Cp", [(16 * 256 * 256, 3), (8 * 128 * 128, 12)])
def test_logit_laplace_decode_mode_writes_only_the_image(n_pix, Cp):
    stats, x = make_inputs(n_pix, Cp, 17)
    xh = run_kernel(stats, x, 0.0, decode=True)
    xt, *_ = run_kernel(stats, x, 1.0 / (n_pix * Cp))
    assert torch.equal(xh, xt)
    assert ((xh.double() - ref64(stats, x)["xh"]).abs() <= 20 * EPS).all()


def test_logit_laplace_sums_are_bit_reproducible():
    stats, x = make_inputs(16 * 256 * 256, 3, 5)
    outs = [run_kernel(stats, x, 1.0 / x.numel()) for _ in range(2)]
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)


def test_logit_laplace_non_finite_stats_stay_in_their_element():
    stats, x = make_inputs(300, 3, 6)
    stats[10, 1] = float("nan")
    stats[20, 4] = float("inf")
    stats[30, 0] = float("-inf")
    xh, ds, *_ = run_kernel(stats, x, 0.5)
    bad = torch.zeros(300, 6, dtype=torch.bool, device=DEV)
    bad[10, 1] = bad[20, 4] = bad[30, 0] = True
    bad_c = bad[:, :3] | bad[:, 3:]          # a subpixel with a non-finite mu or ln b
    assert torch.isfinite(ds[~torch.cat([bad_c, bad_c], -1)]).all()
    assert torch.isfinite(xh[~bad[:, :3]]).all()


def test_logit_laplace_rejects_bad_arguments():
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops
    s = torch.zeros(8, 6, device=DEV)
    x = torch.zeros(8, 3, device=DEV)
    a = torch.zeros(1, device=DEV)
    with pytest.raises(L.DB200Error):
        ops.logit_laplace(s, x, s, x, a, a, 8, 3, float("nan"))
    with pytest.raises(L.DB200Error):
        ops.logit_laplace(s, x, s, x, a, a, 0, 3, 1.0)
    with pytest.raises(L.DB200Error):
        ops.logit_laplace(s, x, s, x, a, a, 8, 0, 1.0)
    sp = L.stream_ptr()
    lib = L.load()
    assert lib.db200_logit_laplace_fwd_bwd(sp, s.data_ptr(), x.data_ptr(), s.data_ptr(), x.data_ptr(), a.data_ptr(),
                                           a.data_ptr(), 8, 3, 1.0, None, 0) != 0         # workspace missing
    assert lib.db200_logit_laplace_fwd_bwd(sp, s.data_ptr(), x.data_ptr(), None, x.data_ptr(), a.data_ptr(),
                                           a.data_ptr(), 8, 3, 1.0, None, 0) != 0         # target without dstats
    assert lib.db200_logit_laplace_fwd_bwd(sp, None, None, None, x.data_ptr(), None, None, 8, 3, 1.0, None, 0) != 0
    assert lib.db200_logit_laplace_workspace_bytes(8, 3) > 0
    assert lib.db200_logit_laplace_workspace_bytes(0, 3) == 0


# ---------------------------------------------------------------------------------------------------------- engine
def _case(convblocks, K, size, B, seed, stack_factor=1, cb_scale=1.0):
    from oracle import vae_logit_laplace as OL
    g = torch.Generator().manual_seed(seed)
    p = OL.init_params(convblocks, K, stack_factor=stack_factor, seed=seed)
    for k in p:
        if k.endswith("/bias"):
            p[k] = torch.randn(p[k].shape, generator=g) * 0.05
    p["codebook/codebook"] = p["codebook/codebook"] * cb_scale
    img = torch.rand(B, size, size, 3, generator=g) * 2 - 1
    hw = size // stack_factor // (2 ** len(convblocks))
    u = torch.rand(B * hw * hw, K, generator=g).clamp_(1e-9, 1.0)
    return p, img, u, hw


def _engine_step(p, img, u, K, size, convblocks, tau, hard, beta, use_bf16=False, stack_factor=1):
    from dalle_mtf_b200.vae_engine import VaeEngine
    eng = VaeEngine(K, size, convblocks, use_bf16=use_bf16, stack_factor=stack_factor, kl=beta is not None,
                    reconstruction_loss="logit_laplace")
    eng.load_params(p)
    eng.zero_grads()
    acc = torch.zeros(3, device=DEV)
    out = eng.forward(img.to(DEV), u.to(DEV), tau, hard, loss_accum=acc[:1], kl_weight=beta,
                      kl_accum=acc[1:2] if beta is not None else None, mse_accum=acc[2:3]).clone()
    eng.backward()
    torch.cuda.synchronize()
    return eng, acc.cpu(), out.cpu(), eng.export_params(eng.grads)


FP32_CASES = [([[2, 32], [2, 64]], 64, 16, 4, True, 1.0, None, 1), ([[2, 32], [2, 64]], 64, 16, 4, False, 0.5, 0.5, 1),
              ([[3, 64], [3, 128], [3, 256]], 512, 32, 8, True, 1.0, None, 1),
              ([[2, 32], [2, 64]], 64, 32, 2, True, 1.0, None, 2), ([[2, 32], [2, 64]], 64, 32, 2, False, 0.7, 0.3, 2)]


@pytest.mark.parametrize("convblocks,K,size,B,hard,tau,beta,s", FP32_CASES)
def test_vae_engine_fp32_logit_laplace_step_matches_oracle(convblocks, K, size, B, hard, tau, beta, s):
    from oracle import vae_logit_laplace as OL
    p, img, u, hw = _case(convblocks, K, size, B, K + size + s, stack_factor=s, cb_scale=8.0 if beta else 1.0)
    uv = u.view(B, hw, hw, K)
    loss, rec, mse, kl, xhat, _, grads = OL.loss_and_grads(p, img, uv, convblocks, tau, hard, stack_factor=s,
                                                           kl_weight=beta)
    eng, acc, out, eg = _engine_step(p, img, u, K, size, convblocks, tau, hard, beta, stack_factor=s)
    assert near(acc[:1], rec) and relfro(acc[2:], mse.reshape(1)) < 1e-4
    if beta is not None:
        assert relfro(acc[1:2], kl.reshape(1)) < 1e-4
        assert near(acc[:1] + beta * acc[1:2], loss)
    assert relfro(out, xhat) < 1e-4
    for k in grads:
        assert relfro(eg[k], grads[k]) < 2e-2, k
    # each mutated oracle is told apart: by the NLL, the image-space output / MSE, or the decoder's gradients
    for m in OL.MUTATIONS:
        _, recm, msem, _, xm, _, gm = OL.loss_and_grads(p, img, uv, convblocks, tau, hard, stack_factor=s,
                                                        kl_weight=beta, mutate=m)
        ok = (near(acc[:1], recm) and relfro(acc[2:], msem.reshape(1)) < 1e-4
              and relfro(out, xm) < 1e-4
              and all(relfro(eg[k], gm[k]) < 2e-2 for k in ("decoder/conv2d/kernel", "decoder/conv2d/bias")))
        assert not ok, m


BF16_CASES = [([[2, 64], [2, 128]], 128, 32, 4, None, 1), ([[2, 64], [2, 128]], 128, 32, 4, 0.5, 1),
              ([[2, 64], [2, 128]], 128, 64, 2, 0.5, 2)]


@pytest.mark.parametrize("cb,K,size,B,beta,s", BF16_CASES)
def test_vae_engine_bf16_logit_laplace_step_within_the_bf16_policy(cb, K, size, B, beta, s):
    from oracle import vae_logit_laplace as OL
    p, img, u, hw = _case(cb, K, size, B, 77 + s, stack_factor=s, cb_scale=8.0 if beta else 1.0)
    uv = u.view(B, hw, hw, K)
    loss, rec, _, _, xhat, _, grads = OL.loss_and_grads(p, img, uv, cb, 1.0, False, stack_factor=s, kl_weight=beta)
    l16, rec16, _, _, x16, _, g16 = OL.loss_and_grads(p, img, uv, cb, 1.0, False, bf16=True, stack_factor=s,
                                                      kl_weight=beta)
    _, acc, out, eg = _engine_step(p, img, u, K, size, cb, 1.0, False, beta, use_bf16=True, stack_factor=s)
    obj = acc[:1] + (beta * acc[1:2] if beta is not None else 0)
    assert abs(obj.item() - loss.item()) <= 1.5 * abs(l16.item() - loss.item()) + 2e-2 * max(abs(loss.item()), 1.0)
    assert relfro(out, xhat) <= 1.5 * relfro(x16, xhat) + 2e-2
    for k in grads:
        e_engine, e_ref = relfro(eg[k], grads[k]), relfro(g16[k], grads[k])
        assert e_engine <= 1.5 * e_ref + 2e-2, (k, e_engine, e_ref)


def test_vae_coco_geometry_k8192_bf16_logit_laplace_kl_step():
    """configs/vae_coco_elb_b200.json geometry: 256 px, [[2,128],[3,256],[5,512]], K = 8192, bf16, soft Gumbel, KL on,
    B = 1."""
    import os
    from oracle import vae_logit_laplace as OL
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    cb, K, size, B, tau, beta = [[2, 128], [3, 256], [5, 512]], 8192, 256, 1, 0.7, 0.034375
    p, img, u, hw = _case(cb, K, size, B, 21, cb_scale=4.0)
    uv = u.view(B, hw, hw, K)
    loss, rec, _, kl, xhat, _, grads = OL.loss_and_grads(p, img, uv, cb, tau, False, kl_weight=beta)
    l16, _, _, _, x16, _, g16 = OL.loss_and_grads(p, img, uv, cb, tau, False, bf16=True, kl_weight=beta)
    _, acc, out, eg = _engine_step(p, img, u, K, size, cb, tau, False, beta, use_bf16=True)
    obj = (acc[:1] + beta * acc[1:2]).item()
    assert abs(obj - loss.item()) <= 1.5 * abs(l16.item() - loss.item()) + 2e-2 * max(abs(loss.item()), 1.0)
    assert relfro(out, xhat) <= 1.5 * relfro(x16, xhat) + 2e-2
    for k in grads:
        e_engine, e_ref = relfro(eg[k], grads[k]), relfro(g16[k], grads[k])
        assert e_engine <= 1.5 * e_ref + 2e-2, (k, e_engine, e_ref)


@pytest.mark.parametrize("use_bf16,s", [(False, 1), (True, 1), (False, 2)])
def test_decode_tokens_equals_the_image_of_a_hard_forward(use_bf16, s):
    from dalle_mtf_b200.vae_engine import VaeEngine
    from oracle import vae_logit_laplace as OL
    cb, K, size, B = [[2, 64], [2, 64]], 64, 16 * s, 3
    p, img, u, hw = _case(cb, K, size, B, 9 + s, stack_factor=s)
    eng = VaeEngine(K, size, cb, use_bf16=use_bf16, stack_factor=s, reconstruction_loss="logit_laplace")
    eng.load_params(p)
    eng.zero_grads()
    out = eng.forward(img.to(DEV), u.to(DEV), 1.0, True).clone()
    codes = eng._b["idx"].view(B, hw * hw).clone()
    dec = eng.decode_tokens(codes + 7, offset=7)
    torch.cuda.synchronize()
    assert torch.equal(dec, out)
    assert (dec.abs() <= 1).all()
    ref = OL.decode(p, codes.view(B, hw, hw).long().cpu(), cb, bf16=use_bf16, stack_factor=s)
    assert relfro(dec, ref) < (2e-2 if use_bf16 else 1e-4)


def _record_ops(monkeypatch):
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


@pytest.mark.parametrize("use_bf16,kl", [(False, None), (True, None), (True, 0.3)])
def test_launch_sequences_without_the_key_and_with_mse(monkeypatch, use_bf16, kl):
    from dalle_mtf_b200.vae_engine import VaeEngine
    from oracle import vae as OV
    cb, K, size, B = [[2, 64], [2, 64]], 64, 16, 2
    p = OV.init_params(cb, K, seed=3)
    img = torch.rand(B, size, size, 3, generator=torch.Generator().manual_seed(3)) * 2 - 1
    u = torch.rand(B * 16, K, generator=torch.Generator().manual_seed(4)).clamp_(1e-9, 1.0)
    seqs = {}
    for key, kw in (("absent", {}), ("mse", {"reconstruction_loss": "mse"})):
        eng = VaeEngine(K, size, cb, use_bf16=use_bf16, kl=kl is not None, **kw)
        eng.load_params(p)
        eng.zero_grads()
        calls = _record_ops(monkeypatch)
        eng.forward(img.to(DEV), u.to(DEV), 1.0, True, kl_weight=kl)
        eng.backward()
        eng.optimizer_step(1e-3, 1)
        decoded = eng.decode_tokens(torch.zeros(B, 16, dtype=torch.int32, device=DEV))
        torch.cuda.synchronize()
        seqs[key] = list(calls)
        monkeypatch.undo()
        assert decoded.shape == (B, size, size, 3)
    assert seqs["absent"] == seqs["mse"]
    assert "logit_laplace" not in seqs["absent"] and seqs["absent"].count("mse_fwd_bwd") == 1


def test_logit_laplace_launch_sequence_swaps_only_the_loss(monkeypatch):
    from dalle_mtf_b200.vae_engine import VaeEngine
    from oracle import vae as OV
    cb, K, size, B = [[2, 64], [2, 64]], 64, 16, 2
    p, img, u, _ = _case(cb, K, size, B, 3)
    seqs = {}
    for key in ("mse", "logit_laplace"):
        eng = VaeEngine(K, size, cb, use_bf16=True, reconstruction_loss=key)
        eng.load_params(p if key == "logit_laplace" else OV.init_params(cb, K, seed=3))
        eng.zero_grads()
        calls = _record_ops(monkeypatch)
        eng.forward(img.to(DEV), u.to(DEV), 1.0, True)
        eng.backward()
        torch.cuda.synchronize()
        seqs[key] = list(calls)
        monkeypatch.undo()
    assert [c if c != "mse_fwd_bwd" else "logit_laplace" for c in seqs["mse"]] == seqs["logit_laplace"]


def test_aux_slots_ride_the_first_bucket():
    from dalle_mtf_b200.vae_engine import VaeEngine
    cb, K, size, B = [[2, 64], [2, 64]], 64, 16, 2
    p, img, u, _ = _case(cb, K, size, B, 4)
    eng = VaeEngine(K, size, cb, kl=True, reconstruction_loss="logit_laplace")
    eng.load_params(p)
    eng.zero_grads()
    ranges = []
    eng.forward(img.to(DEV), u.to(DEV), 1.0, True, kl_weight=0.2)
    eng.backward(on_bucket_ready=lambda s, e: ranges.append((s, e)))
    s, e = ranges[0]
    assert s <= eng.aux_off < eng.aux_off + 2 < e
    torch.cuda.synchronize()
    assert eng.grads[eng.aux_off + 1].item() > 0 and eng.grads[eng.aux_off + 2].item() > 0


# -------------------------------------------------------------------------------------------------------- boundary
def _vae_params(tmp_path, **extra):
    from collections import defaultdict
    d = {"model_type": "vae", "num_tokens": 64, "convblocks": [[2, 64], [2, 64]], "dataset": {"image_size": 16},
         "train_batch_size": 4, "eval_batch_size": 4, "lr": 1e-3, "model_path": str(tmp_path / "vae"),
         "n_channels": 3, "train_gumbel_hard": True, "iterations": 2, "steps_per_checkpoint": 2, "train_steps": 6,
         "reconstruction_loss": "logit_laplace"}
    d.update(extra)
    return defaultdict(lambda: None, d)


@pytest.mark.parametrize("kl", [False, True])
def test_vae_model_fn_matches_oracle_each_step(tmp_path, kl):
    from dalle_mtf_b200.model_fns import EVAL, TRAIN, VAE_LL_KL_PARTS_FORMAT, VAE_LL_PARTS_FORMAT, vae_model_fn
    from oracle import vae_kl as OK
    from oracle import vae_logit_laplace as OL
    extra = {"kl_loss_weight": 0.8, "kl_anneal_steps": 2} if kl else {}
    params = _vae_params(tmp_path, **extra)
    g = torch.Generator().manual_seed(11)
    img = torch.rand(4, 16, 16, 3, generator=g) * 2 - 1
    u = torch.rand(4 * 16, 64, generator=g).clamp_(1e-9, 1.0)
    params["_gumbel_u"] = u.to(DEV)
    spec = vae_model_fn(img, img, TRAIN, params)
    assert spec.loss_parts_format == (VAE_LL_KL_PARTS_FORMAT if kl else VAE_LL_PARTS_FORMAT)
    assert (spec.codebook_usage is not None) == kl
    cb = [[2, 64], [2, 64]]
    for step in range(4):
        p = spec.engine.export_params()
        beta_t = OK.kl_weight(step, params) if kl else None
        loss, rec, mse, klv, _, _, _ = OL.loss_and_grads(p, img, u.view(4, 4, 4, 64), cb, 1.0, True,
                                                         kl_weight=beta_t)
        spec.train_op(img)
        got = float(spec.loss_sum.item()) * spec.loss_scale
        parts = spec.loss_parts.cpu()
        assert near(torch.tensor(got), loss)
        assert parts.numel() == (3 if kl else 2)
        assert near(parts[0], rec) and relfro(parts[1:2], mse.reshape(1)) < 1e-4
        if kl:
            assert relfro(parts[2:], klv.reshape(1)) < 1e-4
    ev = vae_model_fn(img, img, EVAL, params)
    ev.engine.copy_params_from(spec.engine)
    ev.global_step = spec.global_step
    ev.eval_op(img)
    pe = ev.loss_parts.cpu()
    assert pe.numel() == (3 if kl else 2) and torch.isfinite(pe).all()
    got = float(ev.loss_sum.item()) * ev.loss_scale
    assert got == pytest.approx(pe[0].item() + (0.8 * pe[2].item() if kl else 0.0), rel=1e-6, abs=1e-6)


def test_vae_model_fn_checkpoint_round_trip_and_mse_checkpoint_refused(tmp_path):
    from functools import partial
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.input_fns import vae_input_fn
    from dalle_mtf_b200.model_fns import TRAIN, vae_model_fn
    from dalle_mtf_b200.utils import latest_checkpoint, load_checkpoint
    params = _vae_params(tmp_path, kl_loss_weight=0.1)
    est = Estimator(vae_model_fn, params)
    spec = est.train(partial(vae_input_fn, eval=False), max_steps=2)
    saved = spec.state_fn()
    est.close()
    st = load_checkpoint(latest_checkpoint(params["model_path"]))
    assert st["vae/decoder/conv2d/kernel"].shape[-1] == 6
    fresh = vae_model_fn(None, None, TRAIN, params)
    fresh.load_fn(st)
    back = fresh.state_fn()
    assert back.keys() == saved.keys() and all(torch.equal(back[k], saved[k]) for k in saved if k != "global_step")
    est2 = Estimator(vae_model_fn, params)
    spec2 = est2.train(partial(vae_input_fn, eval=False), max_steps=3)
    assert spec2.global_step == 3
    est2.close()
    mse_spec = vae_model_fn(None, None, TRAIN, _vae_params(tmp_path / "m", reconstruction_loss=None))
    with pytest.raises(L.DB200Error, match="decoder/conv2d/kernel"):
        fresh.load_fn(mse_spec.state_fn())
    with pytest.raises(L.DB200Error, match="decoder/conv2d/kernel"):
        mse_spec.load_fn(st)


def test_discrete_vae_model_returns_the_objective():
    from dalle_mtf_b200.models import DiscreteVAE
    from oracle import vae_logit_laplace as OL
    img = torch.rand(2, 16, 16, 3, generator=torch.Generator().manual_seed(0)) * 2 - 1
    for kl in (None, 0.25):
        vae = DiscreteVAE(64, 16, [[2, 64], [2, 64]], kl_loss_weight=kl, reconstruction_loss="logit_laplace")
        loss, out = vae.forward(img, return_recon_loss=True)
        parts = vae.loss_parts.cpu()
        assert parts.numel() == (3 if kl else 2)
        assert loss.item() == pytest.approx(parts[0].item() + (kl * parts[2].item() if kl else 0.0), rel=1e-6, abs=1e-6)
        stats = vae.engine._b["recon_act"].double().cpu()      # fp32 mode: the decoder's output buffer itself
        x = img.double()
        assert parts[0].item() == pytest.approx(OL.nll(stats, x).mean().item(), rel=1e-5, abs=1e-5)
        assert parts[1].item() == pytest.approx(((OL.image(stats) - x) ** 2).mean().item(), rel=1e-4, abs=1e-7)
        assert (out.abs() <= 1).all()
        dec = vae.decode(torch.zeros(2, 16, dtype=torch.int32))
        assert dec.shape == (2, 16, 16, 3) and (dec.abs() <= 1).all()


def _train_vae(tmp_path, **extra):
    from functools import partial
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.input_fns import vae_input_fn
    from dalle_mtf_b200.model_fns import vae_model_fn
    vae_p = _vae_params(tmp_path, steps_per_checkpoint=3, **extra)
    est = Estimator(vae_model_fn, vae_p)
    est.train(partial(vae_input_fn, eval=False), max_steps=3)
    est.close()
    return vae_p


def test_logit_laplace_vae_checkpoint_feeds_dalle_model_fn(tmp_path):
    from collections import defaultdict
    from functools import partial
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.input_fns import dalle_input_fn
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.utils import latest_checkpoint, load_checkpoint
    from oracle import vae as OV
    vae_p = _train_vae(tmp_path, kl_loss_weight=0.1)
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


def test_generate_dalle_decodes_with_a_logit_laplace_vae(tmp_path):
    import json
    import os
    import numpy as np
    import generate_dalle
    from PIL import Image
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.model_fns import load_vae_model
    from dalle_mtf_b200.utils import save_checkpoint
    size, convblocks, K, tv, ts = 16, [[2, 64], [2, 64]], 64, 300, 12
    vae_cfg = {"model_type": "vae", "dataset": {"image_size": size}, "num_tokens": K, "convblocks": convblocks,
               "model_path": str(tmp_path / "vae_run"), "reconstruction_loss": "logit_laplace"}
    dalle_cfg = {"model_type": "dalle", "dataset": {"image_size": size}, "predict_batch_size": 2,
                 "model_path": str(tmp_path / "dalle_run"), "n_embd": 256, "n_layers": 2, "n_heads": 2,
                 "text_vocab_size": tv, "image_vocab_size": K, "text_seq_len": ts,
                 "vae_model": str(tmp_path / "vae.json")}
    (tmp_path / "vae.json").write_text(json.dumps(vae_cfg))
    (tmp_path / "dalle.json").write_text(json.dumps(dalle_cfg))
    params = generate_dalle.load_params(str(tmp_path / "dalle.json"))
    vae, _ = load_vae_model(params, torch.device(DEV))
    assert vae.logit_laplace and vae.out_C == 6
    vae.init_params(4)
    st = {"vae/" + k: v for k, v in vae.export_params().items()}
    st["global_step"] = 7
    save_checkpoint(vae_cfg["model_path"], 7, st)
    hw = size // 4
    eng = DalleEngine(256, 2, 2, tv, K, ts, hw * hw)
    eng.init_params(5)
    st = dict(eng.export_params())
    st["global_step"] = 3
    save_checkpoint(dalle_cfg["model_path"], 3, st)
    np.save(tmp_path / "caps.npy", np.random.default_rng(0).integers(0, tv, (3, ts)).astype(np.int32))
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "dalle.json"), "--out", str(out),
                         "--caption_ids", str(tmp_path / "caps.npy"), "--samples_per_prompt", "2", "--seed", "1"])
    pngs = sorted(p for p in os.listdir(out) if p.endswith(".png"))
    assert len(pngs) == 6
    toks = torch.from_numpy(np.load(out / "tokens.npy")).to(DEV)
    dec = vae.decode_tokens(toks[:, ts:].contiguous(), offset=tv).cpu().numpy()
    want = generate_dalle.to_uint8(dec)
    for j, p in enumerate(pngs):
        assert np.array_equal(np.asarray(Image.open(out / p)), want[j])
