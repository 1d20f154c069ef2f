"""The GELU MLP on the GPU: its two GEMM epilogues against float64, the engines against the oracle, training-step
behaviour and generation.

Epilogues (method of test_dalle_kernels_gpu.py, helpers in float64_bounds.py; U = 2^-24, UTC = 2^-23):
  * z = bf16(x W1 + b1): the STORE bound, b = (K + 8) UTC on absref = |x||W1| + |b1|, plus half a bf16 ulp.
  * h = bf16(gelu(z)) against float64 gelu of the kernel's own z.  The kernel forms v = fma(0.044715 z, z^2, z) (three
    roundings; z and 0.044715 z^3 share a sign, so 3 U relative), t = -2 log2(e) sqrt(2/pi) v (2 U more), 2^t with
    ex2.approx (2^-22 relative, plus the argument's error |t| 5 U ln 2), 1 + 2^t (U), rcp.approx (2^-23) and z s (U):
        eps_h = 4 U |t| + 16 U  relative,   |h - gelu(z)| <= half ulp(|g| (1 + eps_h)) + eps_h |g| + 2^-125 |z|,
    the last term covering the flush to zero where s drops below the fp32 normal range (z below about -10.1).
  * dZ = bf16(acc gelu'(z)) against float64 on the same z: acc carries (K + 8) UTC absref (absref = |dy||W2|^T).
    With f = z c2 (1 + 3 a z^2), gelu' = s + f s (1 - s) carries eps_h (s + |f s (1 - s)|) from s and the products, and
    the second term also carries the error of 1 - s: the subtraction is exact for s >= 1/2 (and U absolute below), but
    it keeps the absolute error eps_h s already in s, so (eps_h s + 2 U) |f| s.  Plus half a bf16 ulp,
    2^-125 |acc| (1 + |f|) for the flush of s to 0 below z ~ -10.1 (gelu' = 0 there) and 2^-126 for products below the
    fp32 normal range.
  * colsum as for RELU_BWD: float64 column sums of the bf16 dZ written, b = (32 + M/32 + 8) U.

Engines: DalleEngine(activation="gelu") against oracle.dalle_gelu.loss_and_grads(activation="gelu"), with
the bounds of test_parity_baseline_gpu.py (loss 1e-3, logits e <= 1.25 e_ref + 2e-3, gradients e <= 1.25 e_ref + 1e-2),
W1 scaled so that z spans the curved part of GELU (std ~2).  The same outputs must fail those bounds against the
oracle with GELU's cubic term removed and against the ReLU oracle.
"""
import ctypes
import gc
import json
import math
import os
import time

import pytest
import torch

import float64_bounds as FB
from float64_bounds import DEV, U, UTC, nan_like

pytestmark = pytest.mark.gpu
TAG = "gelu"
F32, F64, BF16, I16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int16, torch.int32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
A_CUBIC = 0.044715
C2 = 2.0 * math.sqrt(2.0 / math.pi)
T_COEF = 2.0 * math.log2(math.e) * math.sqrt(2.0 / math.pi)

# (name, M rows, d, 4d): the W1 product is [M, d] x [d, 4d], its dgrad [M, d] x [d, 4d]^T.  Training rows are the
# tokens per GPU (dalle_example: 32 x 1280; dalle_coco: 8 x 1280; 12B: 4 x 1280); decode runs 32 rows, guided 64;
# the prefill 3 prompts of 283 positions (not a multiple of the 128-row tile).
SHAPES = [("dalle_example", 40960, 512, 2048), ("dalle_coco", 10240, 1024, 4096), ("12B", 5120, 4096, 16384),
          ("decode32", 32, 512, 2048), ("decode64-guided", 64, 1024, 4096), ("prefill-ragged", 849, 512, 2048)]


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops as O
    L.require_device()
    return O


@pytest.fixture(autouse=True)
def _cost(request):
    gc.collect()
    torch.cuda.synchronize()
    t0 = time.time()
    yield
    torch.cuda.synchronize()
    print(f"[{TAG}] {request.node.name}: {time.time() - t0:.1f} s")


def _bits(t):
    return t.view({F32: I32, BF16: I16}.get(t.dtype, t.dtype))


def gelu64(z, cubic=A_CUBIC):
    """z sigma(2u) = 0.5 z (1 + tanh(u)) without the cancellation of 1 + tanh(u) in the negative tail."""
    return z * torch.sigmoid(C2 * (z + cubic * z ** 3))


def gelu_parts64(z):
    """(s, the derivative's second term, its factor z c2 (1 + 3 a z^2)) in float64."""
    s = torch.sigmoid(C2 * (z + A_CUBIC * z ** 3))
    f = z * C2 * (1.0 + 3.0 * A_CUBIC * z * z)
    return s, f * s * (1.0 - s), f


def eps_h(z):
    return 4 * U * (T_COEF * (z.abs() + A_CUBIC * z.abs() ** 3)) + 16 * U


def check_h(name, h, z):
    """h (bf16, the kernel's) against float64 gelu of the kernel's own z (bf16)."""
    z = z.to(F64)
    g = gelu64(z)
    e = eps_h(z)
    bound = FB.half_ulp_bf16(g.abs() * (1 + e)) + e * g.abs() + 2.0 ** -125 * z.abs()
    bad = (~torch.isfinite(h.to(F64))).sum().item()
    assert bad == 0, f"{name}: {bad} h values are not finite"
    return FB.report(name, ((h.to(F64) - g).abs() / bound.clamp_min(1e-300)).max().item(), TAG)


def check_dz(name, dz, acc, absref, z, K):
    z = z.to(F64)
    s, second, f = gelu_parts64(z)
    d = s + second
    err_d = eps_h(z) * (s + second.abs()) + (eps_h(z) * s + 2 * U) * f.abs() * s
    ref = acc * d
    bound = (K + 8) * UTC * absref * d.abs() + acc.abs() * err_d + 2 * U * ref.abs()
    bound = bound + FB.half_ulp_bf16(ref.abs() + bound) + 2.0 ** -125 * acc.abs() * (1 + f.abs()) + 2.0 ** -126
    bad = (~torch.isfinite(dz.to(F64))).sum().item()
    assert bad == 0, f"{name}: {bad} dZ values are not finite"
    r = (dz.to(F64) - ref).abs() / bound.clamp_min(1e-300)
    i = int(r.flatten().argmax())
    if r.flatten()[i] >= 1:
        at = [t.flatten()[i].item() for t in (z.expand_as(r), acc.expand_as(r), absref.expand_as(r), d.expand_as(r),
                                              dz.to(F64).expand_as(r), ref, bound)]
        print(f"[{TAG}] {name} worst element: z, acc, absref, gelu', got, ref, bound = {at}")
    return FB.report(name, r.max().item(), TAG)


def _operands(M, d, N, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, d, generator=g, device=DEV).to(BF16)                        # LN2 output: unit scale
    w1 = (torch.randn(d, N, generator=g, device=DEV) * (2.0 / math.sqrt(d))).to(BF16)   # z std ~2
    b1 = torch.randn(N, generator=g, device=DEV) * 0.5
    dy = (torch.randn(M, d, generator=g, device=DEV) * 0.01).to(BF16)              # dbranch
    w2 = (torch.randn(N, d, generator=g, device=DEV) * 0.02).to(BF16)
    return x, w1, b1, dy, w2


def _epilogue_case(ops, name, M, d, N, seed):
    x, w1, b1, dy, w2 = _operands(M, d, N, seed)
    h, z = nan_like((M, N), BF16), nan_like((M, N), BF16)
    ops.linear_fwd(x, w1, h, bias=b1, gelu=True, z_out=z)
    h_inf = nan_like((M, N), BF16)
    ops.linear_fwd(x, w1, h_inf, bias=b1, gelu=True)                               # inference: no z output
    base = torch.randn(N, device=DEV)
    colsum = base.clone()
    dz = nan_like((M, N), BF16)
    ops.linear_dgrad(dy, w2, dz, gelu_grad_of=z, colsum=colsum)
    torch.cuda.synchronize()
    assert torch.equal(_bits(h_inf), _bits(h)), f"{name}: h without a z output differs"
    # forward: z within the STORE bound, h against gelu of the kernel's own z
    x64, w164 = x.to(F64), w1.to(F64)
    zref = x64 @ w164 + b1.to(F64)
    zabs = x64.abs() @ w164.abs() + b1.to(F64).abs()
    FB.check(f"{name} z", z, zref, zabs, b=(d + 8) * UTC, bf16_out=True, tag=TAG)
    del zref, zabs, x64, w164
    check_h(f"{name} h", h, z)
    # backward on the stored z: dZ and the fused column sums
    dy64, w264 = dy.to(F64), w2.to(F64)
    acc = dy64 @ w264.T
    absref = dy64.abs() @ w264.abs().T
    check_dz(f"{name} dZ", dz, acc, absref, z, d)
    del acc, absref, dy64, w264
    dz64 = dz.to(F64)
    cref = base.to(F64) + dz64.sum(0)
    FB.check(f"{name} colsum", colsum, cref, base.to(F64).abs() + dz64.abs().sum(0), b=(32 + M / 32 + 8) * U,
             tag=TAG)
    sat = ((z.float() > -1) & (z.float() < 1)).float().mean().item()
    print(f"[{TAG}] {name} M={M} K={d} N={N}: fraction of z in (-1, 1) {sat:.3f}, z range "
          f"[{z.float().min().item():.2f}, {z.float().max().item():.2f}]")


@pytest.mark.parametrize("name,M,d,N", SHAPES, ids=[s[0] for s in SHAPES])
def test_gelu_epilogues_match_float64_at_the_engine_shapes(ops, name, M, d, N):
    _epilogue_case(ops, name, M, d, N, seed=len(name) + M)


def test_gelu_backward_with_sms_reserved(ops):
    """The backward of a data-parallel step runs with SMs reserved for the overlapped all-reduce."""
    with FB.reserved_sms(4):
        _epilogue_case(ops, "dalle_example-4-reserved", 40960, 512, 2048, seed=5)


EDGES = [0.0, -0.0, 1e-30, -1e-30, -3.0, -10.0, -20.0, 1e4, -1e4, float(torch.finfo(BF16).max),
         -float(torch.finfo(BF16).max), float("inf"), float("-inf"), float("nan")]


def test_gelu_epilogues_at_edge_values(ops):
    """Exact z values put in place through the bias (A = 0), and an accumulator of exactly 1 in the backward."""
    n_rep = 16
    vals = torch.tensor(EDGES, dtype=F32, device=DEV)
    N = 64 * math.ceil(len(EDGES) * n_rep / 64)
    bias = vals.repeat(n_rep)
    bias = torch.cat([bias, torch.zeros(N - bias.numel(), device=DEV)])
    M, K = 130, 64
    x = torch.zeros(M, K, dtype=BF16, device=DEV)
    w = torch.randn(K, N, device=DEV).to(BF16)
    h, z = nan_like((M, N), BF16), nan_like((M, N), BF16)
    ops.linear_fwd(x, w, h, bias=bias, gelu=True, z_out=z)
    dy = torch.zeros(M, K, dtype=BF16, device=DEV)
    dy[:, 0] = 1
    w2 = torch.zeros(N, K, dtype=BF16, device=DEV)
    w2[:, 0] = 1
    dz = nan_like((M, N), BF16)
    ops.linear_dgrad(dy, w2, dz, gelu_grad_of=z)
    torch.cuda.synchronize()
    zb = bias.to(BF16)
    assert torch.allclose(z.float(), zb.float().expand(M, N), rtol=0, atol=0, equal_nan=True), "z != bf16(bias)"
    z64 = zb.to(F64).expand(M, N)
    fin = torch.isfinite(z64)
    check_h("edge h (finite z)", h[fin], z[fin])
    assert torch.isfinite(h[fin].float()).all() and torch.isfinite(dz[fin].float()).all()
    zf = z64[0]
    h0, d0 = h[0].float(), dz[0].float()
    assert (h0[zf == float("inf")] == float("inf")).all()
    assert torch.isnan(h0[(zf == float("-inf")) | torch.isnan(zf)]).all()
    assert torch.isnan(d0[~torch.isfinite(zf)]).all()            # as torch's float64 gradient
    big = float(torch.finfo(BF16).max)
    # where sigma is exactly 0 or 1 in fp32, gelu' is exactly 0 or 1 and h is exactly z or (-)0
    for v, dv, hv in ((1e4, 1.0, None), (big, 1.0, None), (-1e4, 0.0, 0.0), (-big, 0.0, 0.0), (-20.0, 0.0, 0.0)):
        sel = zf == float(torch.tensor(v).to(BF16))
        assert (d0[sel] == dv).all(), (v, d0[sel])
        if hv is not None:
            assert (h0[sel] == hv).all(), (v, h0[sel])
        else:
            assert (h0[sel] == zf[sel].float()).all(), (v, h0[sel])
    # finite z: dZ = bf16(gelu'(z)) within the bound, and exactly the float64 value's rounding at 0 and 1e-30
    ok = fin[0]
    check_dz("edge dZ (finite z)", dz[:, ok], torch.ones_like(z64[:, ok]), torch.ones_like(z64[:, ok]), z[:, ok], 1)
    for v in (0.0, -0.0, 1e-30, -1e-30):
        sel = zf == float(torch.tensor(v).to(BF16))
        assert (d0[sel] == 0.5).all() and (h0[sel].abs() <= 1e-30).all()
    # -3: the negative tail keeps its relative accuracy (tanh.approx would be ~20 % off here)
    sel = zf == -3.0
    g3 = gelu64(torch.tensor(-3.0, dtype=F64)).item()
    assert ((h0[sel] - g3).abs() <= 2 ** -7 * abs(g3)).all(), (h0[sel], g3)
    print(f"[{TAG}] edge values {EDGES}: h / gelu' rules hold")


def test_gelu_entry_points_reject_bad_arguments(ops):
    from dalle_mtf_b200 import lib as L
    x = torch.zeros(128, 64, dtype=BF16, device=DEV)
    w = torch.zeros(64, 128, dtype=BF16, device=DEV)
    out = torch.empty(128, 128, dtype=BF16, device=DEV)
    z = torch.empty(128, 136, dtype=BF16, device=DEV)
    ops.linear_fwd(x, w, out, gelu=True, z_out=z[:, :128])                          # ldz = 136: fine
    with pytest.raises(L.DB200Error):
        ops.linear_fwd(x, w, out, gelu=True, z_out=torch.empty(128, 132, dtype=BF16, device=DEV)[:, :128])
    with pytest.raises(L.DB200Error):       # operand majors: the GELU store needs a k-major A and an mn-major B
        ops.gemm(x, w.T.contiguous(), out, 128, 128, 64, a_mn=False, b_mn=False, gelu="fwd")
    with pytest.raises(L.DB200Error):       # the backward needs aux = z
        ops.gemm(x, w.T.contiguous(), out, 128, 128, 64, mode=L.EPI_RELU_BWD, gelu="bwd")
    with pytest.raises(L.DB200Error):
        ops.gemm(x, w, out, 128, 128, 64, a_mn=False, b_mn=True, gelu="fwd", residual=out)
    with pytest.raises(L.DB200Error):
        ops.linear_fwd(x, w, out, gelu=True, relu=True)
    with pytest.raises(L.DB200Error):
        ops.linear_dgrad(out, w, x, relu_mask_of=out, gelu_grad_of=out)
    lib = L.load()
    e = L.GemmEpilogue()
    e.mode, e.alpha = L.EPI_STORE, 1.0
    assert lib.db200_gemm_bf16_gelu(None, L.ptr(x), 0, 64, L.ptr(w), 1, 128, L.ptr(out), 128, 128, 128, 64,
                                    None, None, 0) != 0
    e.mode = L.EPI_CE_GRAD
    assert lib.db200_gemm_bf16_gelu_bwd(None, L.ptr(out), 0, 128, L.ptr(w), 0, 128, L.ptr(x), 64, 128, 64, 128,
                                        ctypes.byref(e)) != 0
    e.mode = L.EPI_RELU_BWD
    e.colsum = L.ptr(torch.zeros(128, device=DEV))
    e.aux, e.ldaux = L.ptr(out), 128
    assert lib.db200_gemm_workspace_bytes(1000, 128, 64, ctypes.byref(e)) == 8 * 4 * 128 * 4
    torch.cuda.synchronize()


# ================================================================================================ engines vs oracle
def relfro(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _params(cfg, seed):
    from oracle import dalle as O
    p = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in p:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            p[k] = torch.randn(p[k].shape, generator=g) * 0.02
        if k.endswith("/g"):
            p[k] = 1 + torch.randn(p[k].shape, generator=g) * 0.05
        if k.endswith("mlp_linear_1/kernel"):        # z = LN2(x) W1 + b1 with std ~2: the curved part of GELU
            p[k] = p[k] * (100.0 / math.sqrt(cfg.n_embd))
        if k.endswith("mlp_linear_1/bias"):
            p[k] = torch.randn(p[k].shape, generator=g) * 0.5
    return p


def _violations(loss, rows, lg, grads, o32, o16):
    """The parity rules of test_parity_baseline_gpu.py; returns the list of the ones broken."""
    loss32, rows32, logits32, g32 = o32
    _, _, logits16, g16 = o16
    out = []
    lr = abs(loss - loss32.item()) / abs(loss32.item())
    if lr > 1e-3:
        out.append(("loss", lr))
    re = relfro(rows, rows32)
    if re > 5e-3:
        out.append(("loss_rows", re))
    e, er = relfro(lg, logits32), relfro(logits16, logits32)
    if not (e <= 1.25 * er + 2e-3 and e <= 2e-2):
        out.append(("logits", e, er))
    for k in g32:
        ee, er = relfro(grads[k], g32[k]), relfro(g16[k], g32[k])
        if ee > 1.25 * er + 1e-2:
            out.append((k, ee, er))
    return out


def _engine_case(name, d, L, H, tv, iv, ts, isl, B, seed, recompute=False, attention_types=None, kernel=5,
                 dropout=None, mutations=False):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    from oracle import dalle_gelu as OG
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    layers = None
    if attention_types is not None:
        import conv_oracle as OC
        cfg = OC.ConvConfig(d, L, H, tv, iv, ts, isl, attention_types=tuple(attention_types),
                            local_attention_radius=256, conv_attention_kernel=kernel)
        layers = OC
    else:
        cfg = O.DalleConfig(d, L, H, tv, iv, ts, isl)
    spec = None if dropout is None else (dropout[0], dropout[1], 3, 0)
    params = _params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 2)
    text = torch.randint(0, tv - 1, (B, ts), generator=g)
    img = torch.randint(0, iv, (B, isl), generator=g)
    tokens = O.assemble_tokens(text, img, tv)

    def oracle(act, mutate=None):
        return [OG.loss_and_grads(params, tokens, cfg, spec, bf16=bf, activation=act, mutate=mutate, layers=layers)
                for bf in (False, True)]

    o32, o16 = oracle("gelu")
    kw = {}
    if dropout is not None:
        kw = dict(dropout=dropout[0], dropout_seed=dropout[1])
    eng = DalleEngine(d, L, H, tv, iv, ts, isl, recompute_grad=recompute, attention_types=attention_types,
                      conv_attention_kernel=kernel, activation="gelu", **kw)
    eng.load_params(params)
    tok = tokens.to(I32).to(DEV)
    T = tokens.numel()
    eng.zero_grads()
    acc = eng.forward(tok, step=3 if dropout is not None else None)
    eng.backward(1.0 / T)
    torch.cuda.synchronize()
    loss = acc.item() / T
    rows = eng._bufs["loss_rows"].float().cpu().view(B, -1)
    grads = {k: v.clone() for k, v in eng.export_params(eng.grads).items()}
    if dropout is not None:     # the training forward's logits: replay the dropout forward through the output GEMM
        lg = torch.empty(T, eng.Vpad, dtype=F32, device=DEV)
        eng.forward(tok, loss_accum=torch.zeros(1, device=DEV), step=3)
        from dalle_mtf_b200 import ops as OPS
        OPS.gemm(eng._bufs["hf"], eng.W("wout"), lg, T, eng.Vpad, d, a_mn=False, b_mn=True, bias=eng.P("bout"))
        lg = lg.view(B, -1, eng.Vpad)[:, :, :eng.V].cpu()
    else:
        lg = eng.logits(tok).float().cpu()
    bad = _violations(loss, rows, lg, grads, o32, o16)
    print(f"[{TAG}] {name}: loss {loss:.6f} oracle {o32[0].item():.6f}, logits relfro {relfro(lg, o32[2]):.2e} "
          f"(reference bf16 policy {relfro(o16[2], o32[2]):.2e}), violations {bad}")
    assert not bad, bad
    if mutations:
        for act, mut in (("gelu", "gelu_no_cubic"), ("relu", None)):
            m32, m16 = oracle(act, mut)
            vb = _violations(loss, rows, lg, grads, m32, m16)
            print(f"[{TAG}] {name} against the {mut or act} oracle: {len(vb)} rules broken, e.g. {vb[:3]}")
            assert vb, f"{name}: the engine also matches the {mut or act} oracle"
    return eng


def test_one_layer_engine_matches_the_gelu_oracle_and_not_the_mutants():
    _engine_case("one layer d256", 256, 1, 2, 300, 64, 24, 40, 2, seed=21, mutations=True)


def test_engine_with_dropout_matches_the_gelu_oracle_and_not_the_mutants():
    _engine_case("d256 L2 dropout", 256, 2, 2, 300, 64, 24, 40, 2, seed=22, dropout=((0.1, 0.1, 0.1), 7),
                 mutations=True)


def test_dalle_example_geometry_matches_the_gelu_oracle():
    _engine_case("EX d512 L6 H4 S1280 V50771 B1", 512, 6, 4, 50258, 512, 256, 1024, 1, seed=23)


def test_dalle_coco_geometry_recompute_with_a_sparse_schedule_matches_the_gelu_oracle():
    _engine_case("CO d1024 L3 H16 S1280 B1 recompute row/conv/global", 1024, 3, 16, 50258, 512, 256, 1024, 1,
                 seed=24, recompute=True, attention_types=["axial_row", "conv", "global"], kernel=5)


# ================================================================================================ call sets
def _record_gemms(monkeypatch):
    from dalle_mtf_b200 import ops as O
    calls = []
    real = O.gemm

    def gemm(*a, **k):
        calls.append((k.get("mode", 0), k.get("gelu"), bool(k.get("relu")), k.get("z") is not None, a[3]))
        return real(*a, **k)
    monkeypatch.setattr(O, "gemm", gemm)
    return calls


def test_call_sets(monkeypatch):
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.sampling import DalleSampler
    calls = _record_gemms(monkeypatch)
    g = torch.Generator().manual_seed(4)
    tok = torch.randint(0, 299, (2, 64), generator=g).to(I32).to(DEV)
    for act, recompute in (("gelu", False), ("gelu", True), ("relu", False)):
        Ly = 3
        eng = DalleEngine(256, Ly, 2, 300, 64, 24, 40, activation=act, recompute_grad=recompute)
        eng.init_params(1)
        calls.clear()
        eng.zero_grads()
        eng.forward(tok)
        eng.backward(1.0)
        torch.cuda.synchronize()
        fwd = [c for c in calls if c[1] == "fwd"]
        bwd = [c for c in calls if c[1] == "bwd"]
        relu_store = [c for c in calls if c[2]]
        relu_bwd = [c for c in calls if c[0] == L.EPI_RELU_BWD and c[1] is None]
        if act == "gelu":
            # every layer: the GELU store with z (twice per layer under recompute_grad) and the GELU backward
            assert len(fwd) == Ly * (2 if recompute else 1) and all(c[3] for c in fwd), calls
            assert len(bwd) == Ly and not relu_store and not relu_bwd, calls
        else:
            assert not fwd and not bwd and len(relu_store) == Ly and len(relu_bwd) == Ly, calls
        smp = DalleSampler(eng)
        calls.clear()
        text = torch.randint(0, 299, (2, 24), generator=g).to(I32).to(DEV)
        smp.generate(text, temperature=0.0)
        smp.generate_graphed(text, temperature=0.0)
        smp.complete(text, image_prefix=torch.randint(0, 64, (2, 5), generator=g).to(DEV))
        torch.cuda.synchronize()
        w1 = [c for c in calls if c[1] == "fwd" or c[2]]
        assert w1 and all((c[1] == "fwd") == (act == "gelu") and not c[3] for c in w1), calls
        print(f"[{TAG}] call set {act} recompute={recompute}: {len(fwd)} GELU stores, {len(bwd)} GELU backwards; "
              f"sampler / prefill W1 products {len(w1)}, none with a z output")


# ================================================================================================ training steps
def test_two_gelu_steps_are_bit_identical():
    from dalle_mtf_b200.dalle_engine import DalleEngine
    g = torch.Generator().manual_seed(6)
    tok = torch.randint(0, 299, (4, 64), generator=g).to(I32).to(DEV)
    outs = []
    for _ in range(2):
        eng = DalleEngine(256, 2, 2, 300, 64, 24, 40, activation="gelu", dropout=(0.1, 0.1, 0.1), dropout_seed=2)
        eng.init_params(3)
        for step in range(2):
            eng.zero_grads()
            eng.forward(tok, step=step)
            eng.backward(1.0 / tok.numel())
            eng.optimizer_step(1e-3)
        torch.cuda.synchronize()
        outs.append((eng.grads.clone(), eng.master.clone(), eng.shadow.clone()))
    for a, b in zip(*outs):
        assert torch.equal(_bits(a), _bits(b))


def test_gelu_ranks_equal_micro_batches_bitwise(monkeypatch, tmp_path):
    import test_data_parallel_gpu as DP
    rec = DP._Rec(monkeypatch)
    extra = {"activation_function": "gelu", "recompute_grad": True}
    for W, B in ((2, 12), (3, 12)):
        make = lambda **kw: DP._dalle_params(tmp_path, extra, train_batch_size=B, **kw)     # noqa: E731
        p = make()
        feats, caps = DP._dalle_data(p, B, seed=W)
        ref, n, aux_off = DP._dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * DP._seq_len(p)),
                                              feats, caps, W)
        assert next(iter(rec.fwd), None) is None
        group, chk, (n_r, aux_r) = DP._dalle_ranks(rec, make, feats, caps, W, ref)
        assert (n_r, aux_r) == (n, aux_off)
        chk.assert_clean()
        print(f"[{TAG}] GELU W={W} B={B}: {chk.bitwise} tensors bitwise equal to one rank with {W} micro-batches")


def test_model_fn_steps_from_the_gelu_config_run_and_log():
    """Three training steps of configs/dalle_example_gelu_b200.json through the Estimator (the loop train_dalle.py
    runs), logging every step: each step writes its log line with a finite loss near ln V at initialisation."""
    import itertools
    import re
    from collections import defaultdict
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.model_fns import dalle_model_fn
    with open(os.path.join(ROOT, "configs", "dalle_example_gelu_b200.json")) as f:
        cfg = json.load(f)
    assert cfg["activation_function"] == "gelu"
    p = defaultdict(lambda: None, cfg)
    # the configuration's transformer at a small batch, with a random-init stand-in of its tokenizer; no checkpoints
    p.update(train_batch_size=2, model_path=None, iterations=1, vae_random_init=True, dataset={"image_size": 64},
             vae_params=defaultdict(lambda: None, {"model_type": "vae", "num_tokens": 512, "convblocks": [[1, 32]],
                                                   "dataset": {"image_size": 64}}))
    g = torch.Generator().manual_seed(1)
    feats = torch.rand(2, 64, 64, 3, generator=g) * 2 - 1
    caps = torch.randint(0, 50257, (2, 256), generator=g)

    class Log:
        lines = []

        def info(self, msg):
            self.lines.append(msg)

    log = Log()
    spec = Estimator(dalle_model_fn, p, logger=log).train(lambda params: itertools.repeat((feats, caps)), max_steps=3)
    assert spec.engine.activation == "gelu" and "z1" in spec.engine._bufs["layers"][0]
    steps = [re.match(r"step (\d+) loss (\S+) ", ln) for ln in log.lines]
    got = [(int(m.group(1)), float(m.group(2))) for m in steps if m]
    print(f"[{TAG}] dalle_example_gelu_b200 (d512 L6, B=2, 32x32 tokens) log: {log.lines}")
    V = cfg["text_vocab_size"] + cfg["image_vocab_size"] + 1
    assert [s for s, _ in got] == [1, 2, 3], log.lines
    assert all(math.isfinite(v) and abs(v - math.log(V)) < 1.5 for _, v in got), got


# ================================================================================================ generation
def _gelu_model(d=256, L=2, H=2, tv=300, iv=64, ts=24, isl=40, seed=3):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    cfg = O.DalleConfig(d, L, H, tv, iv, ts, isl)
    params = _params(cfg, seed)
    for k in params:
        if "wte" in k or "linear_out" in k:
            params[k] = params[k] * 4                       # sharper logits: clear arg-maxima
    eng = DalleEngine(d, L, H, tv, iv, ts, isl, activation="gelu")
    eng.load_params(params)
    return eng, cfg, params


def test_greedy_generation_equals_the_full_forward_argmax_and_replay_equals_eager():
    from dalle_mtf_b200.sampling import DalleSampler
    eng, cfg, params = _gelu_model()
    tv, iv, ts, S = 300, 64, 24, 64
    g = torch.Generator().manual_seed(9)
    text = torch.randint(0, tv, (3, ts), generator=g).to(I32).to(DEV)
    smp = DalleSampler(eng)
    toks, step_logits = smp.generate(text, temperature=0, return_logits=True)
    graphed = smp.generate_graphed(text, temperature=0)
    torch.cuda.synchronize()
    assert torch.equal(graphed, toks)
    img = graphed[:, ts:]
    full = eng.logits(graphed)
    dec = torch.stack(step_logits, 1)
    e = relfro(dec, full[:, :S - 1])
    assert e < 2e-2, e
    rng = full[:, ts - 1:S - 1, tv:tv + iv]
    top2 = rng.topk(2, -1).values
    clear = (top2[..., 0] - top2[..., 1]) > 0.05 * rng.abs().max()
    same = (rng.argmax(-1) + tv) == img
    assert (same | ~clear).all() and clear.float().mean() > 0.2 and same.float().mean() > 0.8
    print(f"[{TAG}] greedy GELU generation: replay == eager, {same.float().mean().item():.3f} of the tokens are the "
          f"full forward's argmax (all of the clear ones), decode-vs-full logits relfro {e:.2e}")


def test_prefill_logits_at_position_p_match_decoding():
    from dalle_mtf_b200.sampling import DalleSampler
    eng, cfg, params = _gelu_model()
    tv, ts = 300, 24
    g = torch.Generator().manual_seed(10)
    text = torch.randint(0, tv, (2, ts), generator=g).to(I32).to(DEV)
    smp = DalleSampler(eng)
    toks, step_logits = smp.generate(text, temperature=0, return_logits=True)
    for n in (1, 7):
        P = ts + n
        kc = [torch.zeros(2, eng.S, eng.H, eng.dh, dtype=BF16, device=DEV) for _ in range(eng.L)]
        vc = [torch.zeros_like(c) for c in kc]
        lg = eng.prefill(toks[:, :P].contiguous(), kc, vc)[:, :eng.V]
        e = relfro(lg, step_logits[P - 1])
        print(f"[{TAG}] prefill P={P}: position-P logits vs decoding relfro {e:.2e}")
        assert e < 2e-2, e
