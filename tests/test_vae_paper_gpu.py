"""GPU tests of the DALL-E paper's discrete-VAE network (architecture "dalle_paper"): the K11p kernels against
float64, the engine against oracle/vae_paper.py, and the model boundary.

Kernel bounds, eps = 2^-24 (f32), u = 2^-8 (the bf16 rounding of a stored output, half an ulp is 2^-9 relative):
  * conv7x7_in_fwd: y = b + sum over 49 C taps of x w, f32 FMAs in a fixed order: a running f32 sum of n = 49 C + 1
    terms is within n eps sum |terms| of the exact one (each FMA rounds once); the stored bf16 output adds u |y|.
  * conv7x7_in_wgrad: each dw element is a sum over the M pixels: a lane group sums its M / (4 splits) pixels in order,
    4 lane groups, then the splits in order, then the add into dw: n = ceil(M / (4 splits)) + 4 + splits + 1 roundings,
    |err| <= n eps sum |x dy| + eps |dw|.
  * maxpool fwd / bwd, upsample fwd: exact (selection and copies).
  * upsample bwd: ((a + b) + c) + d in f32: 3 eps sum |.|, plus u |s| for a bf16 output.
  * residual_gain: fma(gain, r, id) rounded once in f32: eps |v|, plus u |v| for bf16.
Outputs are NaN-filled with guard elements behind them; inputs include bf16 values with many exact ties, odd batch and
spatial sizes.

Engine: fp32 at small geometries against the oracle at the tolerances of tests/test_vae_logit_laplace_gpu.py's fp32
step; bf16 at the paper geometry against the oracle's bf16 policy (the oracle runs on the GPU in f32 with TF32 off);
mutated oracles must fail.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24
U = 2.0 ** -8


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def relfro(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def near(a, b, tol=1e-4):
    a, b = float(a.reshape(-1)[0]), float(b.reshape(-1)[0])
    return abs(a - b) <= tol * max(abs(b), 1.0)


def nan_buf(shape, dtype, guard=64):
    n = math.prod(shape)
    buf = torch.full((n + guard,), float("nan"), dtype=dtype, device=DEV)
    return buf, buf[:n].view(*shape)


def guards_ok(buf, n):
    return bool(torch.isnan(buf[n:].float()).all())


def tie_tensor(shape, dtype, seed):
    """Values on a coarse grid (many exact ties, exact in bf16), a slice of continuous values."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randint(-4, 5, shape, generator=g, device=DEV).float() * 0.25
    x.view(-1)[::5] = torch.randn(x.view(-1)[::5].shape, generator=g, device=DEV)
    return x.to(dtype)


# ---------------------------------------------------------------------------------------------------------- kernels
def conv7_ref(x, w, b):
    xd = x.double().permute(0, 3, 1, 2)
    wd = w.double().permute(3, 2, 0, 1)
    y = torch.nn.functional.conv2d(xd, wd, b.double(), padding=3).permute(0, 2, 3, 1)
    mag = torch.nn.functional.conv2d(xd.abs(), wd.abs(), b.double().abs(), padding=3).permute(0, 2, 3, 1)
    return y, mag


@pytest.mark.parametrize("N,H,W,C,Cout,dtype", [(3, 17, 23, 3, 64, torch.bfloat16), (1, 32, 32, 3, 256, torch.bfloat16),
                                                 (2, 9, 40, 3, 72, torch.float32), (1, 8, 8, 1, 8, torch.float32),
                                                 (2, 13, 7, 4, 136, torch.bfloat16)])
def test_conv7x7_in_fwd_against_float64(N, H, W, C, Cout, dtype):
    from dalle_mtf_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(N * H + C)
    x = torch.rand(N, H, W, C, generator=g, device=DEV) * 2 - 1
    w = torch.randn(7, 7, C, Cout, generator=g, device=DEV) / math.sqrt(49 * C)
    b = torch.randn(Cout, generator=g, device=DEV) * 0.1
    buf, y = nan_buf((N, H, W, Cout), dtype)
    ops.conv7x7_in_fwd(x, w, b, y)
    torch.cuda.synchronize()
    assert guards_ok(buf, y.numel())
    ref, mag = conv7_ref(x, w, b)
    bound = (49 * C + 1) * EPS * mag + (U if dtype == torch.bfloat16 else 0) * ref.abs() + 1e-30
    assert ((y.double() - ref).abs() <= bound).all()


@pytest.mark.parametrize("N,H,W,C,Cout,dtype", [(3, 17, 23, 3, 64, torch.bfloat16), (2, 9, 40, 3, 72, torch.float32),
                                                 (1, 64, 64, 3, 256, torch.bfloat16), (2, 13, 7, 4, 136, torch.float32)])
def test_conv7x7_in_wgrad_against_float64(N, H, W, C, Cout, dtype):
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(H * W + Cout)
    x = torch.rand(N, H, W, C, generator=g, device=DEV) * 2 - 1
    dy = tie_tensor((N, H, W, Cout), dtype, 5)
    base_w = torch.randn(7, 7, C, Cout, generator=g, device=DEV)
    base_b = torch.randn(Cout, generator=g, device=DEV)
    dw, db = base_w.clone(), base_b.clone()
    ops.conv7x7_in_wgrad(x, dy, dw, db)
    torch.cuda.synchronize()
    xd, dyd = x.double(), dy.double()
    xp = torch.nn.functional.pad(xd, (0, 0, 3, 3, 3, 3))
    ref = torch.zeros(7, 7, C, Cout, dtype=torch.float64, device=DEV)
    mag = torch.zeros_like(ref)
    for kh in range(7):
        for kw in range(7):
            patch = xp[:, kh:kh + H, kw:kw + W, :].reshape(-1, C)
            ref[kh, kw] = patch.t() @ dyd.reshape(-1, Cout)
            mag[kh, kw] = patch.abs().t() @ dyd.abs().reshape(-1, Cout)
    M = N * H * W
    splits = L.load().db200_conv7x7_in_wgrad_workspace_bytes(N, H, W, C, Cout) // 4 // (49 * C * Cout + Cout)
    n = -(-M // (4 * splits)) + 4 + splits + 1
    exp_w = base_w.double() + ref
    assert ((dw.double() - exp_w).abs() <= n * EPS * (mag + base_w.double().abs()) + EPS * exp_w.abs()).all()
    exp_b = base_b.double() + dyd.reshape(-1, Cout).sum(0)
    mag_b = dyd.abs().reshape(-1, Cout).sum(0) + base_b.double().abs()
    assert ((db.double() - exp_b).abs() <= n * EPS * mag_b + EPS * exp_b.abs()).all()
    # bit-reproducible
    dw2, db2 = base_w.clone(), base_b.clone()
    ops.conv7x7_in_wgrad(x, dy, dw2, db2)
    assert torch.equal(dw, dw2) and torch.equal(db, db2)
    # no bias gradient requested
    dw3 = base_w.clone()
    ops.conv7x7_in_wgrad(x, dy, dw3, None)
    assert torch.equal(dw3, dw)


def pool_ref(x):
    """(values, first-maximum index 0..3 in raster order) of every 2x2 window, float64 on the GPU."""
    N, H, W, C = x.shape
    win = x.double().reshape(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(N, H // 2, W // 2, C, 4)
    m = win.max(-1).values
    first = (win == m.unsqueeze(-1)).to(torch.int64).argmax(-1)
    return m, first


def unwindow(g4, shape):
    N, H, W, C = shape
    return g4.reshape(N, H // 2, W // 2, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(N, H, W, C)


@pytest.mark.parametrize("N,H,W,C,dtype", [(3, 6, 10, 5, torch.bfloat16), (1, 32, 32, 256, torch.bfloat16),
                                           (5, 2, 14, 7, torch.float32), (2, 64, 64, 64, torch.bfloat16)])
def test_maxpool_fwd_bwd_exact_with_ties(N, H, W, C, dtype):
    from dalle_mtf_b200 import ops
    from oracle import vae_paper as P
    x = tie_tensor((N, H, W, C), dtype, N + C)
    dy = tie_tensor((N, H // 2, W // 2, C), dtype, 7) + 3
    ybuf, y = nan_buf((N, H // 2, W // 2, C), dtype)
    dbuf, dx = nan_buf((N, H, W, C), dtype)
    ops.maxpool2x2_fwd(x, y)
    ops.maxpool2x2_bwd(x, dy, dx)
    torch.cuda.synchronize()
    assert guards_ok(ybuf, y.numel()) and guards_ok(dbuf, dx.numel())
    m, first = pool_ref(x)
    assert torch.equal(y.double(), m)
    ties = (x.double().reshape(N, H // 2, 2, W // 2, 2, C).amax((2, 4)) == m)
    assert ties.all()
    onehot = torch.nn.functional.one_hot(first, 4).double() * dy.double().unsqueeze(-1)
    assert torch.equal(dx.double(), unwindow(onehot, x.shape))
    # the oracle's rule (autograd through oracle/vae_paper.max_pool) and its last-maximum mutation
    xr = x.float().cpu().requires_grad_(True)
    (P.max_pool(xr) * dy.float().cpu()).sum().backward()
    assert torch.equal(dx.float().cpu(), xr.grad)
    win = x.double().reshape(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(N, H // 2, W // 2, C, 4)
    assert ((win == m.unsqueeze(-1)).sum(-1) > 1).any(), "the inputs must contain tied windows"
    xl = x.float().cpu().requires_grad_(True)
    (P.max_pool(xl, "tie_last") * dy.float().cpu()).sum().backward()
    assert not torch.equal(dx.float().cpu(), xl.grad)


def test_maxpool_past_2_31_elements():
    """x of 4 x 512 x 512 x 2056 bf16 = 2.16e9 elements; the last image is checked against the reference."""
    from dalle_mtf_b200 import ops
    N, H, W, C = 4, 512, 512, 2056
    assert N * H * W * C > 2 ** 31
    x = torch.empty(N, H, W, C, dtype=torch.bfloat16, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(1)
    for n in range(N):
        x[n] = (torch.randint(-3, 4, (H, W, C), generator=g, device=DEV).float() * 0.5).to(torch.bfloat16)
    y = torch.full((N, H // 2, W // 2, C), float("nan"), dtype=torch.bfloat16, device=DEV)
    ops.maxpool2x2_fwd(x, y)
    dy = torch.ones_like(y)
    dx = torch.full_like(x, float("nan"))
    ops.maxpool2x2_bwd(x, dy, dx)
    torch.cuda.synchronize()
    m, first = pool_ref(x[-1:])
    assert torch.equal(y[-1:].double(), m)
    assert torch.equal(dx[-1:].double(), unwindow(torch.nn.functional.one_hot(first, 4).double(), (1, H, W, C)))
    assert not torch.isnan(y).any() and not torch.isnan(dx).any()


@pytest.mark.parametrize("N,H,W,C,dtype", [(3, 5, 7, 5, torch.bfloat16), (2, 32, 32, 256, torch.bfloat16),
                                           (1, 3, 9, 6, torch.float32)])
def test_upsample_fwd_exact_bwd_against_float64(N, H, W, C, dtype):
    from dalle_mtf_b200 import ops
    x = tie_tensor((N, H, W, C), dtype, 3)
    ybuf, y = nan_buf((N, 2 * H, 2 * W, C), dtype)
    ops.upsample2x_fwd(x, y)
    dy = torch.randn(N, 2 * H, 2 * W, C, generator=torch.Generator(device=DEV).manual_seed(2), device=DEV).to(dtype)
    dbuf, dx = nan_buf((N, H, W, C), dtype)
    ops.upsample2x_bwd(dy, dx)
    torch.cuda.synchronize()
    assert guards_ok(ybuf, y.numel()) and guards_ok(dbuf, dx.numel())
    assert torch.equal(y, x.repeat_interleave(2, 1).repeat_interleave(2, 2))
    blocks = dy.double().reshape(N, H, 2, W, 2, C)
    ref, mag = blocks.sum((2, 4)), blocks.abs().sum((2, 4))
    bound = 3 * EPS * mag + (U if dtype == torch.bfloat16 else 0) * ref.abs()
    assert ((dx.double() - ref).abs() <= bound).all()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_residual_gain_against_float64(dtype):
    from dalle_mtf_b200 import ops
    n = 3 * 1001
    r, idv, mask = (tie_tensor((n,), dtype, s) for s in (1, 2, 3))
    for gain, use_id, use_mask in ((1 / 64, True, False), (0.3, False, False), (1.0, False, True), (1 / 9, True, True)):
        ybuf, y = nan_buf((n,), dtype)
        abuf, a = nan_buf((n,), dtype)
        ops.residual_gain(r, gain, id=idv if use_id else None, mask=mask if use_mask else None, y=y, relu_y=a)
        torch.cuda.synchronize()
        assert guards_ok(ybuf, n) and guards_ok(abuf, n)
        g32 = torch.tensor(gain, dtype=torch.float32).item()     # the kernel's gain is the f32 value
        v = g32 * r.double() + (idv.double() if use_id else 0)
        if use_mask:
            v = torch.where(mask.double() > 0, v, torch.zeros_like(v))
        bound = (EPS + (U if dtype == torch.bfloat16 else 0)) * v.abs()
        assert ((y.double() - v).abs() <= bound).all()
        assert torch.equal(a, torch.relu(y))
    # in place, ReLU only
    z = r.clone()
    ops.residual_gain(z, 1.0, y=z)
    out = torch.empty_like(r)
    ops.residual_gain(r, 1.0, relu_y=out)
    assert torch.equal(z, r) and torch.equal(out, torch.relu(r))


def test_k11p_rejects_what_it_does_not_cover():
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops
    x = torch.zeros(1, 6, 6, 5, device=DEV)
    with pytest.raises(L.DB200Error):
        ops.conv7x7_in_fwd(x, torch.zeros(7, 7, 5, 64, device=DEV), None, torch.zeros(1, 6, 6, 64, device=DEV))
    with pytest.raises(L.DB200Error):
        ops.conv7x7_in_fwd(x[..., :3].contiguous(), torch.zeros(7, 7, 3, 12, device=DEV), None,
                           torch.zeros(1, 6, 6, 12, device=DEV))
    with pytest.raises(L.DB200Error):
        ops.maxpool2x2_fwd(torch.zeros(1, 5, 6, 8, device=DEV), torch.zeros(1, 2, 3, 8, device=DEV))
    with pytest.raises(L.DB200Error):
        ops.residual_gain(torch.zeros(8, device=DEV), 1.0)
    with pytest.raises(L.DB200Error):
        ops.residual_gain(torch.zeros(8, device=DEV), float("nan"), y=torch.zeros(8, device=DEV))
    assert L.load().db200_conv7x7_in_wgrad_workspace_bytes(1, 8, 8, 5, 64) == 0


# ---------------------------------------------------------------------------------------------------------- engine
def _case(K, size, B, seed, ll, geo, dev="cpu", bias=0.05):
    from oracle import vae_paper as P
    g = torch.Generator().manual_seed(seed)
    p = P.init_params(K, logit_laplace=ll, seed=seed, **geo)
    for k in p:
        if k.endswith("/bias"):
            p[k] = torch.randn(p[k].shape, generator=g) * bias
    img = torch.rand(B, size, size, 3, generator=g) * 2 - 1
    hw = size // 2 ** (geo["group_count"] - 1)
    u = torch.rand(B * hw * hw, K, generator=g).clamp_(1e-9, 1.0)
    if dev != "cpu":
        p = {k: v.to(dev) for k, v in p.items()}
    return p, img.to(dev), u.to(dev), hw


def _engine(K, size, geo, ll, kl, use_bf16):
    from dalle_mtf_b200.vae_paper_engine import PaperVaeEngine
    return PaperVaeEngine(K, size, use_bf16=use_bf16, kl=kl, reconstruction_loss="logit_laplace" if ll else "mse",
                          **geo)


def _engine_step(eng, p, img, u, tau, hard, beta):
    eng.load_params(p)
    eng.zero_grads()
    acc = torch.zeros(3, device=DEV)
    out = eng.forward(img.to(DEV), u.to(DEV), tau, hard, loss_accum=acc[:1], kl_weight=beta,
                      kl_accum=acc[1:2] if beta is not None else None,
                      mse_accum=acc[2:3] if eng.logit_laplace else None).clone()
    logits = eng._b["logits"].clone()
    eng.backward()
    torch.cuda.synchronize()
    return acc.cpu(), out.cpu(), logits.cpu(), eng.export_params(eng.grads)


def _oracle(p, img, u, hw, geo, tau, hard, ll, beta, bf16=False, mutate=None):
    from oracle import vae_paper as P
    B, K = img.shape[0], u.shape[-1]
    return P.loss_and_grads(p, img, u.view(B, hw, hw, K), temperature=tau, hard=hard, bf16=bf16, logit_laplace=ll,
                            kl_weight=beta, mutate=mutate, **geo)


SMALL = [  # (geo, K, size, B, ll, beta, hard, tau)
    (dict(n_hid=64, n_blk_per_group=1, group_count=2, n_init=64), 512, 32, 3, False, None, True, 1.0),
    (dict(n_hid=64, n_blk_per_group=2, group_count=3, n_init=64), 512, 32, 2, True, 0.5, False, 0.7),
    (dict(n_hid=64, n_blk_per_group=1, group_count=4, n_init=128), 512, 32, 2, True, None, True, 1.0),
    (dict(n_hid=72, n_blk_per_group=2, group_count=2, n_init=40), 96, 18, 3, False, 0.3, False, 1.0),
]


@pytest.mark.parametrize("geo,K,size,B,ll,beta,hard,tau", SMALL)
def test_paper_engine_fp32_step_matches_oracle(geo, K, size, B, ll, beta, hard, tau):
    p, img, u, hw = _case(K, size, B, K + size + B, ll, geo)
    loss, rec, mse, kl, out_ref, logits_ref, grads = _oracle(p, img, u, hw, geo, tau, hard, ll, beta)
    eng = _engine(K, size, geo, ll, beta is not None, False)
    assert eng.image_seq_len == hw * hw and eng.n_params() == sum(v.numel() for v in p.values())
    acc, out, logits, eg = _engine_step(eng, p, img, u, tau, hard, beta)
    assert relfro(logits, logits_ref.reshape(-1, K)) < 1e-5
    assert near(acc[:1], rec)
    if ll:
        assert relfro(acc[2:], mse.reshape(1)) < 1e-4
    if beta is not None:
        assert relfro(acc[1:2], kl.reshape(1)) < 1e-4
    assert relfro(out, out_ref) < 1e-4
    for k in grads:
        assert relfro(eg[k], grads[k]) < 2e-2, k
    # every mutated oracle is told apart, by the logits, the output or a gradient ("tie_last" needs tied pool windows,
    # which continuous f32 activations do not have: test_mutations_fail_on_tied_pool_windows)
    from oracle import vae_paper as P
    for m in P.MUTATIONS:
        if m == "tie_last":
            continue
        _, recm, _, _, om, lm, gm = _oracle(p, img, u, hw, geo, tau, hard, ll, beta, mutate=m)
        ok = (relfro(logits, lm.reshape(-1, K)) < 1e-5 and near(acc[:1], recm) and relfro(out, om) < 1e-4
              and all(relfro(eg[k], gm[k]) < 2e-2 for k in grads))
        assert not ok, m


def test_mutations_fail_on_tied_pool_windows():
    """The tie rule shows when the pooled activations tie: a network whose encoder input conv is zero but for a bias
    makes every window of group 1's output tie exactly (in fp32 and bf16 alike)."""
    geo = dict(n_hid=64, n_blk_per_group=1, group_count=2, n_init=64)
    K, size, B = 64, 16, 2
    p, img, u, hw = _case(K, size, B, 5, False, geo)
    p["encoder/input/kernel"] = torch.zeros_like(p["encoder/input/kernel"])
    p["encoder/input/kernel"][3, 3, 0] = 1.0          # x0 = img channel 0 + bias, tied wherever the image ties
    for j in (1, 2, 3, 4):                            # the block adds a constant: the ties reach the pool
        p[f"encoder/group_1/block_1/res_path/conv_{j}/kernel"].zero_()
    img = (torch.randint(0, 2, img.shape, generator=torch.Generator().manual_seed(1)).float() * 0.5)
    loss, _, _, _, out_ref, _, grads = _oracle(p, img, u, hw, geo, 1.0, True, False, None)
    _, _, _, _, _, _, gl = _oracle(p, img, u, hw, geo, 1.0, True, False, None, mutate="tie_last")
    eng = _engine(K, size, geo, False, False, False)
    acc, out, _, eg = _engine_step(eng, p, img, u, 1.0, True, None)
    k = "encoder/input/kernel"
    assert relfro(eg[k], grads[k]) < 1e-4
    assert relfro(eg[k], gl[k]) > 1e-3


def test_paper_geometry_bf16_step_within_the_bf16_policy():
    """256^2, n_hid 256, 2 blocks per group, 4 groups, n_init 128, K 8192, 2 images, logit-Laplace, KL on, soft Gumbel:
    the engine's error against the f32 oracle is within 1.5x the oracle's own bf16-policy error (+ 2e-2)."""
    geo = dict(n_hid=256, n_blk_per_group=2, group_count=4, n_init=128)
    K, size, B, tau, beta = 8192, 256, 2, 0.7, 0.034375
    p, img, u, hw = _case(K, size, B, 21, True, geo, dev=DEV)
    loss, rec, _, kl, xhat, logits_ref, grads = _oracle(p, img, u, hw, geo, tau, False, True, beta)
    l16, _, _, _, x16, lg16, g16 = _oracle(p, img, u, hw, geo, tau, False, True, beta, bf16=True)
    eng = _engine(K, size, geo, True, True, True)
    acc, out, logits, eg = _engine_step(eng, p, img, u, tau, False, beta)
    obj = (acc[:1] + beta * acc[1:2]).item()
    assert abs(obj - loss.item()) <= 1.5 * abs(l16.item() - loss.item()) + 2e-2 * max(abs(loss.item()), 1.0)
    assert relfro(logits, logits_ref.reshape(-1, K)) <= 1.5 * relfro(lg16, logits_ref) + 2e-2
    assert relfro(out, xhat) <= 1.5 * relfro(x16, xhat) + 2e-2
    worst = 0.0
    for k in grads:
        e_engine, e_ref = relfro(eg[k], grads[k]), relfro(g16[k], grads[k])
        assert e_engine <= 1.5 * e_ref + 2e-2, (k, e_engine, e_ref)
        worst = max(worst, e_engine)
    print(f"paper geometry bf16: worst gradient rel-fro {worst:.3g}")


@pytest.mark.parametrize("ll", [False, True])
def test_paper_bf16_mse_and_hard_gumbel_small(ll):
    geo = dict(n_hid=64, n_blk_per_group=2, group_count=3, n_init=64)
    K, size, B = 256, 32, 3
    p, img, u, hw = _case(K, size, B, 8, ll, geo)
    loss, _, _, _, o32, _, grads = _oracle(p, img, u, hw, geo, 1.0, True, ll, None)
    l16, _, _, _, o16, _, g16 = _oracle(p, img, u, hw, geo, 1.0, True, ll, None, bf16=True)
    eng = _engine(K, size, geo, ll, False, True)
    acc, out, _, eg = _engine_step(eng, p, img, u, 1.0, True, None)
    assert abs(acc[0].item() - loss.item()) <= 1.5 * abs(l16.item() - loss.item()) + 2e-2 * max(abs(loss.item()), 1)
    assert relfro(out, o32) <= 1.5 * relfro(o16, o32) + 2e-2
    for k in grads:
        assert relfro(eg[k], grads[k]) <= 1.5 * relfro(g16[k], grads[k]) + 2e-2, k


@pytest.mark.parametrize("use_bf16", [False, True])
def test_buckets_are_disjoint_cover_the_buffer_tail_first(use_bf16):
    geo = dict(n_hid=64, n_blk_per_group=1, group_count=2, n_init=64)
    K, size, B = 64, 16, 2
    p, img, u, _ = _case(K, size, B, 4, True, geo)
    eng = _engine(K, size, geo, True, True, use_bf16)
    eng.load_params(p)
    eng.zero_grads()
    ranges = []
    eng.forward(img.to(DEV), u.to(DEV), 1.0, True, kl_weight=0.2)
    eng.backward(on_bucket_ready=lambda s, e: ranges.append((s, e)))
    torch.cuda.synchronize()
    assert len(ranges) == 2 and ranges[0][0] > ranges[1][0]
    assert sorted(ranges) == [(0, ranges[0][0]), (ranges[0][0], eng.grads.numel())]
    assert eng.grads[eng.aux_off + 1].item() > 0 and eng.grads[eng.aux_off + 2].item() > 0


@pytest.mark.parametrize("use_bf16", [False, True])
def test_decode_tokens_equals_the_output_of_a_hard_forward(use_bf16):
    from oracle import vae_paper as P
    geo = dict(n_hid=64, n_blk_per_group=1, group_count=3, n_init=64)
    K, size, B = 64, 32, 3
    p, img, u, hw = _case(K, size, B, 9, True, geo)
    eng = _engine(K, size, geo, True, False, use_bf16)
    eng.load_params(p)
    eng.zero_grads()
    out = eng.forward(img.to(DEV), u.to(DEV), 1.0, True).clone()
    codes = eng._b["idx"].view(B, hw * hw).clone()
    dec = eng.decode_tokens(codes + 7, offset=7)
    toks = eng.encode_tokens(img.to(DEV)).clone()
    torch.cuda.synchronize()
    assert torch.equal(dec, out)
    ref = P.decode(p, codes.view(B, hw, hw).long().cpu(), bf16=use_bf16, logit_laplace=True, **geo)
    assert relfro(dec, ref) < (2e-2 if use_bf16 else 1e-4)
    logits = P.encoder(p, img, bf16=use_bf16, **{k: geo[k] for k in ("n_hid", "n_blk_per_group", "group_count")})
    logits = logits.reshape(-1, K)
    got = eng.encode_logits(img.to(DEV)).cpu()
    tol = 2 * (got - logits).abs().max().item()      # rows whose top two logits lie within the engine's deviation
    top2 = logits.topk(2, -1).values
    clear = (top2[:, 0] - top2[:, 1]) > tol
    assert clear.float().mean() > 0.5
    assert torch.equal(toks.cpu().reshape(-1)[clear], logits.argmax(-1)[clear].to(torch.int32))


# -------------------------------------------------------------------------------------------------------- boundary
def _vae_params(tmp_path, **extra):
    from collections import defaultdict
    d = {"model_type": "vae", "num_tokens": 64, "architecture": "dalle_paper", "n_hid": 64, "n_blk_per_group": 1,
         "group_count": 2, "n_init": 64, "dataset": {"image_size": 16}, "train_batch_size": 6, "eval_batch_size": 6,
         "lr": 1e-3, "model_path": str(tmp_path / "vae"), "n_channels": 3, "train_gumbel_hard": True,
         "iterations": 2, "steps_per_checkpoint": 2, "train_steps": 6, "reconstruction_loss": "logit_laplace"}
    d.update(extra)
    return defaultdict(lambda: None, d)


GEO = dict(n_hid=64, n_blk_per_group=1, group_count=2, n_init=64)


def test_vae_model_fn_steps_match_the_oracle(tmp_path):
    from dalle_mtf_b200.model_fns import TRAIN, vae_model_fn
    from oracle import vae_kl as OK
    params = _vae_params(tmp_path, kl_loss_weight=0.5, kl_anneal_steps=2)
    g = torch.Generator().manual_seed(11)
    img = torch.rand(6, 16, 16, 3, generator=g) * 2 - 1
    u = torch.rand(6 * 64, 64, generator=g).clamp_(1e-9, 1.0)
    params["_gumbel_u"] = u.to(DEV)
    spec = vae_model_fn(img, img, TRAIN, params)
    assert type(spec.engine).__name__ == "PaperVaeEngine"
    for step in range(3):
        p = spec.engine.export_params()
        loss, rec, mse, klv, _, _, _ = _oracle(p, img, u, 8, GEO, 1.0, True, True, OK.kl_weight(step, params))
        spec.train_op(img)
        assert near(torch.tensor(float(spec.loss_sum.item()) * spec.loss_scale), loss)
        parts = spec.loss_parts.cpu()
        assert near(parts[0], rec) and relfro(parts[2:], klv.reshape(1)) < 1e-4


@pytest.mark.parametrize("W", [2, 3])
def test_vae_model_fn_ranks_match_the_oracle_of_the_global_batch(tmp_path, W):
    from rank_group import RankGroup
    from dalle_mtf_b200.model_fns import TRAIN, vae_model_fn
    B = 6
    g = torch.Generator().manual_seed(17 + W)
    img = torch.rand(B, 16, 16, 3, generator=g) * 2 - 1
    u = torch.rand(B * 64, 64, generator=g).clamp_(1e-9, 1.0)
    b, rows = B // W, B // W * 64
    group = RankGroup(W)
    shared = {}

    def fn(rank, dp):
        pr = _vae_params(tmp_path, model_path=None, kl_loss_weight=0.3)
        pr["_dp"] = dp
        pr["_gumbel_u"] = u[rank * rows:(rank + 1) * rows].to(DEV)
        x = img[rank * b:(rank + 1) * b]
        spec = vae_model_fn(x, x, TRAIN, pr)
        p = spec.engine.export_params()
        spec.train_op(x)
        full = torch.zeros_like(spec.engine.grads)
        for red in group.last_reduce:
            off, numel, _, _ = red["sig"]
            full[off:off + numel] = red["result"]
        shared[rank] = (p, float(spec.loss_sum.item()) * spec.loss_scale, spec.engine.export_params(full * (1.0 / W)),
                        spec.engine.export_params())
        return 0

    group.run(fn)
    p, obj, grad, after = shared[0]
    loss, _, _, _, _, _, grads = _oracle(p, img, u, 8, GEO, 1.0, True, True, 0.3)
    assert near(torch.tensor(obj), loss)
    for k in grads:
        assert relfro(grad[k], grads[k]) < 2e-2, k
    for r in range(1, W):
        assert shared[r][1] == obj and all(torch.equal(shared[r][3][k], after[k]) for k in after)


def test_save_load_and_resume_continue_the_run(tmp_path):
    """The checkpoint holds vae/<name>, /Adam and /Adam_1 of the paper's parameters and restores them bit for bit;
    a run resumed from it continues the uninterrupted run (same noise and batch).  The continued state equals it to
    rounding: the direct convolutions' weight gradients add their pixel splits with float atomics."""
    from functools import partial
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.input_fns import vae_input_fn
    from dalle_mtf_b200.model_fns import TRAIN, vae_model_fn
    from dalle_mtf_b200.utils import latest_checkpoint, load_checkpoint
    a = _vae_params(tmp_path / "a", steps_per_checkpoint=2, use_bf16=True, kl_loss_weight=0.1)
    est = Estimator(vae_model_fn, a)
    spec = est.train(partial(vae_input_fn, eval=False), max_steps=2)
    est.close()
    st = load_checkpoint(latest_checkpoint(a["model_path"]))
    assert {k for k in st if k.endswith("/Adam")} and {k for k in st if k.endswith("/Adam_1")}
    assert "vae/encoder/input/kernel" in st and "vae/decoder/input/kernel" in st and "vae/codebook/codebook" not in st
    fresh = vae_model_fn(None, None, TRAIN, a)
    fresh.load_fn(st)
    back, saved = fresh.state_fn(), spec.state_fn()
    assert back.keys() == saved.keys() and all(torch.equal(back[k], saved[k]) for k in saved if k != "global_step")
    # fixed noise and batch: 2 + 2 steps through a checkpoint against 4 straight steps
    g = torch.Generator().manual_seed(3)
    img = torch.rand(6, 16, 16, 3, generator=g) * 2 - 1
    u = torch.rand(6 * 64, 64, generator=g).clamp_(1e-9, 1.0).to(DEV)
    runs = {}
    for name, split in (("straight", None), ("resumed", 2)):
        pr = _vae_params(tmp_path / name, use_bf16=True, kl_loss_weight=0.1, kl_anneal_steps=3)
        pr["_gumbel_u"] = u
        sp = vae_model_fn(img, img, TRAIN, pr)
        for step in range(4):
            if step == split:
                ck = sp.state_fn()
                sp = vae_model_fn(img, img, TRAIN, pr)
                sp.load_fn(ck)
                assert sp.global_step == split
            sp.train_op(img)
        runs[name] = sp.state_fn()
    a, b = runs["straight"], runs["resumed"]
    assert a["global_step"] == b["global_step"] == 4
    for k in a:
        if k != "global_step":
            assert relfro(b[k], a[k]) < 1e-5, k


def test_dalle_model_fn_tokens_from_a_paper_vae(tmp_path):
    from collections import defaultdict
    from functools import partial
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.input_fns import dalle_input_fn, vae_input_fn
    from dalle_mtf_b200.model_fns import dalle_model_fn, vae_model_fn
    from dalle_mtf_b200.utils import latest_checkpoint, load_checkpoint
    from oracle import vae_paper as P
    vae_p = _vae_params(tmp_path, steps_per_checkpoint=2, train_batch_size=4)
    est = Estimator(vae_model_fn, vae_p)
    est.train(partial(vae_input_fn, eval=False), max_steps=2)
    est.close()
    st = load_checkpoint(latest_checkpoint(vae_p["model_path"]))
    w = {k[4:]: v for k, v in st.items() if k.startswith("vae/") and not k.endswith(("/Adam", "/Adam_1"))}
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
    toks = spec.assemble(img, cap).cpu().long()[:, 12:] - 300
    est2.close()
    logits = P.encoder(w, torch.as_tensor(img).float(), n_hid=64, n_blk_per_group=1, group_count=2).reshape(-1, 64)
    top2 = logits.topk(2, -1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-4 * top2[:, 0].abs().clamp_min(1)
    assert clear.float().mean() > 0.9
    assert torch.equal(toks.reshape(-1)[clear], logits.argmax(-1)[clear])


def test_generate_dalle_decodes_through_the_paper_decoder(tmp_path):
    import json
    import os
    import numpy as np
    import generate_dalle
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.model_fns import load_vae_model
    from dalle_mtf_b200.utils import save_checkpoint
    size, K, tv, ts = 16, 64, 300, 12
    vae_cfg = {"model_type": "vae", "dataset": {"image_size": size}, "num_tokens": K, "architecture": "dalle_paper",
               "n_hid": 64, "n_blk_per_group": 1, "group_count": 2, "n_init": 64,
               "model_path": str(tmp_path / "vae_run"), "reconstruction_loss": "logit_laplace"}
    dalle_cfg = {"model_type": "dalle", "dataset": {"image_size": size}, "predict_batch_size": 2,
                 "model_path": str(tmp_path / "dalle_run"), "n_embd": 256, "n_layers": 2, "n_heads": 2,
                 "text_vocab_size": tv, "image_vocab_size": K, "text_seq_len": ts,
                 "vae_model": str(tmp_path / "vae.json")}
    (tmp_path / "vae.json").write_text(json.dumps(vae_cfg))
    (tmp_path / "dalle.json").write_text(json.dumps(dalle_cfg))
    params = generate_dalle.load_params(str(tmp_path / "dalle.json"))
    assert generate_dalle.token_grid_side(params) == 8
    vae, _ = load_vae_model(params, torch.device(DEV))
    assert type(vae).__name__ == "PaperVaeEngine" and vae.image_seq_len == 64
    vae.init_params(4)
    st = {"vae/" + k: v for k, v in vae.export_params().items()}
    st["global_step"] = 7
    save_checkpoint(vae_cfg["model_path"], 7, st)
    eng = DalleEngine(256, 2, 2, tv, K, ts, 64)
    eng.init_params(5)
    st = dict(eng.export_params())
    st["global_step"] = 3
    save_checkpoint(dalle_cfg["model_path"], 3, st)
    np.save(tmp_path / "caps.npy", np.random.default_rng(0).integers(0, tv, (3, ts)).astype(np.int32))
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "dalle.json"), "--out", str(out),
                         "--caption_ids", str(tmp_path / "caps.npy"), "--samples_per_prompt", "1", "--seed", "1"])
    pngs = sorted(f for f in os.listdir(out) if f.endswith(".png"))
    assert len(pngs) == 3
    from PIL import Image
    toks = torch.from_numpy(np.load(out / "tokens.npy")).to(DEV)
    dec = vae.decode_tokens(toks[:, ts:].contiguous(), offset=tv).cpu().numpy()
    want = generate_dalle.to_uint8(dec)
    for j, f in enumerate(pngs):
        assert np.array_equal(np.asarray(Image.open(out / f)), want[j])


def test_discrete_vae_model_with_the_paper_architecture():
    from dalle_mtf_b200.models import DiscreteVAE
    img = torch.rand(2, 16, 16, 3, generator=torch.Generator().manual_seed(0)) * 2 - 1
    vae = DiscreteVAE(64, 16, architecture="dalle_paper", n_hid=64, n_blk_per_group=1, group_count=2, n_init=64,
                      kl_loss_weight=0.25, reconstruction_loss="logit_laplace")
    loss, out = vae.forward(img, return_recon_loss=True)
    parts = vae.loss_parts.cpu()
    assert loss.item() == pytest.approx(parts[0].item() + 0.25 * parts[2].item(), rel=1e-6, abs=1e-6)
    assert out.shape == (2, 16, 16, 3) and (out.abs() <= 1).all()
    dec = vae.decode(torch.zeros(2, 64, dtype=torch.int32))
    assert dec.shape == (2, 16, 16, 3)
    with pytest.raises(ValueError, match="convblocks"):
        DiscreteVAE(64, 16, [[2, 64]], architecture="dalle_paper")
