"""The gated MLP on the GPU: its two GEMM epilogues against float64, the engines against the oracle, training-step
behaviour, checkpoints, generation and launches.

Epilogues (method of test_gelu_gpu.py, helpers in float64_bounds.py; U = 2^-24, UTC = 2^-23, K = d the W1 product's
contraction, the dgrad's contraction d as well):
  * z = [zv | zg] = bf16(x W1 + b1): the STORE bound, (K + 8) UTC on absref = |x||W1| + |b1|, plus half a bf16 ulp.
  * h, from the kernel's own z.  ReGLU: h = bf16(zv (zg > 0 ? zg : 0)) evaluated in float32, bit for bit.  GEGLU: the
    kernel's a = bf16(gelu(zg)) is within B_a = half ulp(|g| (1 + eps_h)) + eps_h |g| + 2^-125 |zg| of g = float64
    gelu(zg) (test_gelu_gpu.py's h bound, eps_h = 4 U |t| + 16 U), and zv a is exact in fp32, so
        |h - zv g| <= |zv| B_a + half ulp(|zv| (|g| + B_a)).
  * dz = [dzv | dzg] against float64 on the same z, with dh = acc in fp32 carrying E = (K + 8) UTC absref
    (absref = |dy||W2|^T):
        dzv = bf16(dh a):            ref acc g;  bound E |g| + (|acc| + E) B_a + U |ref|, plus half a bf16 ulp.
        dzg = bf16((dh act'(zg)) zv): ref acc act'(zg) zv with ReGLU's act' = [zg > 0] (bound (E + 2 U |acc|) |zv|
                                      where zg > 0, exactly 0 elsewhere) and GEGLU's gelu' (test_gelu_gpu.py's error
                                      err_d of gelu', so E |d| |zv| + |acc| err_d |zv| + 2 U |ref| + 2^-125 |acc| (1 +
                                      |f|) |zv| + 2^-126), plus half a bf16 ulp.
  * colsum over all 2N columns as for RELU_BWD: float64 column sums of the bf16 dz written, b = (32 + M/32 + 8) U.

Engines: DalleEngine(gated_mlp=True) against oracle.dalle_glu.loss_and_grads with the bounds of
test_parity_baseline_gpu.py (loss 1e-3, logits e <= 1.25 e_ref + 2e-3, gradients e <= 1.25 e_ref + 1e-2), the gate
half of W1 scaled so that zg spans the curved part of GELU.  The same outputs must fail those bounds against the
"swap" and "shift64" mutants and against the ungated oracle.
"""
import ctypes
import gc
import math
import time

import pytest
import torch

import float64_bounds as FB
import test_gelu_gpu as GE
from float64_bounds import DEV, U, UTC, nan_like
from test_loss_weights_gpu import _engine, _step, _tiny_params, relfro

pytestmark = pytest.mark.gpu
TAG = "gated_mlp"
F32, F64, BF16, I16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int16, torch.int32
ACTS = ("relu", "gelu")
SHAPES = GE.SHAPES        # (name, M, d, 4d): dalle_example, dalle_coco, 12B, decode 32 / 64, ragged prefill 849


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


def relu_gate32(zv, zg):
    """ReGLU's h in float32 from the kernel's z: bf16(zv (zg > 0 ? zg : 0))."""
    zv, zg = zv.float(), zg.float()
    return (zv * torch.where(zg > 0, zg, torch.zeros_like(zg))).to(BF16)


def gate_bound(zg):
    """(g, B_a): float64 gelu(zg) and the bound on the kernel's a = bf16(gelu(zg))."""
    zg = zg.to(F64)
    g = GE.gelu64(zg)
    e = GE.eps_h(zg)
    return g, FB.half_ulp_bf16(g.abs() * (1 + e)) + e * g.abs() + 2.0 ** -125 * zg.abs()


def check_h(name, act, h, z):
    n = h.shape[1]
    zv, zg = z[:, :n], z[:, n:]
    if act == "relu":
        want = relu_gate32(zv, zg)
        same = torch.equal(_bits(h), _bits(want))
        print(f"[{TAG}] {name}: ReGLU h {'equals' if same else 'differs from'} bf16(zv relu(zg)) bit for bit")
        assert same, name
        return 0.0
    g, ba = gate_bound(zg)
    zv = zv.to(F64)
    ref = zv * g
    bound = zv.abs() * ba + FB.half_ulp_bf16(zv.abs() * (g.abs() + ba))
    bad = (~torch.isfinite(h.to(F64))).sum().item()
    assert bad == 0, f"{name}: {bad} h values are not finite"
    return FB.report(name, ((h.to(F64) - ref).abs() / bound.clamp_min(1e-300)).max().item(), TAG)


def check_dz(name, act, dz, acc, absref, z, K):
    n = acc.shape[1]
    zv, zg = z[:, :n].to(F64), z[:, n:].to(F64)
    E = (K + 8) * UTC * absref
    if act == "relu":
        g, ba = torch.where(zg > 0, zg, torch.zeros_like(zg)), torch.zeros_like(zg)
        pos = zg > 0
        ref_g = torch.where(pos, acc * zv, torch.zeros_like(acc))
        bnd_g = torch.where(pos, (E + 2 * U * acc.abs()) * zv.abs(), torch.zeros_like(acc))
    else:
        g, ba = gate_bound(zg)
        s, second, f = GE.gelu_parts64(zg)
        dd = s + second
        err_d = GE.eps_h(zg) * (s + second.abs()) + (GE.eps_h(zg) * s + 2 * U) * f.abs() * s
        ref_g = acc * dd * zv
        bnd_g = E * dd.abs() * zv.abs() + acc.abs() * err_d * zv.abs() + 2 * U * ref_g.abs() + \
            2.0 ** -125 * acc.abs() * (1 + f.abs()) * zv.abs() + 2.0 ** -126
    ref_v = acc * g
    bnd_v = E * g.abs() + (acc.abs() + E) * ba + U * ref_v.abs() + 2.0 ** -126
    r = 0.0
    for part, got, ref, bnd in (("dzv", dz[:, :n], ref_v, bnd_v), ("dzg", dz[:, n:], ref_g, bnd_g)):
        bad = (~torch.isfinite(got.to(F64))).sum().item()
        assert bad == 0, f"{name} {part}: {bad} values are not finite"
        bound = bnd + FB.half_ulp_bf16(ref.abs() + bnd)
        ratio = (got.to(F64) - ref).abs() / bound.clamp_min(1e-300)
        r = max(r, FB.report(f"{name} {part}", ratio.max().item(), TAG))
    return r


def _operands(M, d, N, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, d, generator=g, device=DEV).to(BF16)                             # LN2 output: unit scale
    w1 = (torch.randn(d, 2 * N, generator=g, device=DEV) * (2.0 / math.sqrt(d))).to(BF16)   # z std ~2
    b1 = torch.randn(2 * N, generator=g, device=DEV) * 0.5
    dy = (torch.randn(M, d, generator=g, device=DEV) * 0.01).to(BF16)                   # dbranch
    w2 = (torch.randn(N, d, generator=g, device=DEV) * 0.02).to(BF16)
    return x, w1, b1, dy, w2


def glu_case(ops, name, M, d, N, act, seed):
    """Both GLU epilogues at [M, d] x [d, 2N] -> h [M, N] and [M, d] x [N, d]^T -> dz [M, 2N], checked in float64."""
    x, w1, b1, dy, w2 = _operands(M, d, N, seed)
    h, z = nan_like((M, N), BF16), nan_like((M, 2 * N), BF16)
    ops.linear_fwd(x, w1, h, bias=b1, glu=act, z_out=z)
    h_inf = nan_like((M, N), BF16)
    ops.linear_fwd(x, w1, h_inf, bias=b1, glu=act)                                      # inference: no z output
    base = torch.randn(2 * N, device=DEV)
    colsum = base.clone()
    dz = nan_like((M, 2 * N), BF16)
    ops.linear_dgrad(dy, w2, dz, glu_grad_of=z, glu=act, colsum=colsum)
    torch.cuda.synchronize()
    assert torch.equal(_bits(h_inf), _bits(h)), f"{name}: h without a z output differs"
    x64, w164 = x.to(F64), w1.to(F64)
    zref = x64 @ w164 + b1.to(F64)
    zabs = x64.abs() @ w164.abs() + b1.to(F64).abs()
    r = FB.check(f"{name} {act} z", z, zref, zabs, b=(d + 8) * UTC, bf16_out=True, tag=TAG)
    del zref, zabs, x64, w164
    r = max(r, check_h(f"{name} {act} h", act, h, z))
    dy64, w264 = dy.to(F64), w2.to(F64)
    acc = dy64 @ w264.T
    absref = dy64.abs() @ w264.abs().T
    r = max(r, check_dz(f"{name} {act}", act, dz, acc, absref, z, d))
    del acc, absref, dy64, w264
    dz64 = dz.to(F64)
    cref = base.to(F64) + dz64.sum(0)
    r = max(r, FB.check(f"{name} {act} colsum", colsum, cref, base.to(F64).abs() + dz64.abs().sum(0),
                        b=(32 + M / 32 + 8) * U, tag=TAG))
    return r


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("name,M,d,N", SHAPES, ids=[s[0] for s in SHAPES])
def test_glu_epilogues_match_float64_at_the_engine_shapes(ops, name, M, d, N, act):
    glu_case(ops, name, M, d, N, act, seed=len(name) + M)


@pytest.mark.parametrize("act", ACTS)
def test_glu_epilogues_at_ragged_rows_and_with_sms_reserved(ops, act):
    glu_case(ops, "ragged-M 333", 333, 256, 192, act, seed=3)          # N = 3 x 64: an odd number of 64-column tiles
    with FB.reserved_sms(4):
        glu_case(ops, "dalle_example-4-reserved", 40960, 512, 2048, act, seed=5)


def _same(a, b):
    """Equal element for element, NaN matching NaN."""
    a, b = a.float(), b.float()
    return bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def test_glu_epilogues_at_edge_values(ops):
    """Exact z values put in place through the bias (A = 0): every edge value of test_gelu_gpu.py meets every edge
    value as (zv, zg), and an accumulator of exactly 1 in the backward.  ReGLU's h, dzv and dzg are their float32
    expressions bit for bit (NaN for NaN); GEGLU's are within their bounds where both halves are moderate, and NaN or
    inf propagate as torch's float arithmetic propagates them."""
    edges = GE.EDGES
    n_e = len(edges)
    N = 64 * math.ceil(n_e * n_e / 64)
    vals = torch.tensor(edges, dtype=F32, device=DEV)
    zv = torch.zeros(N, device=DEV)
    zg = torch.zeros(N, device=DEV)
    zv[:n_e * n_e] = vals.repeat_interleave(n_e)
    zg[:n_e * n_e] = vals.repeat(n_e)
    bias = torch.cat([zv, zg])
    M, K = 130, 64
    x = torch.zeros(M, K, dtype=BF16, device=DEV)
    w = torch.randn(K, 2 * N, device=DEV).to(BF16)
    dy = torch.zeros(M, K, dtype=BF16, device=DEV)
    dy[:, 0] = 1
    w2 = torch.zeros(N, K, dtype=BF16, device=DEV)
    w2[:, 0] = 1
    zb = bias.to(BF16)
    v, gt = zb[:N].float(), zb[N:].float()
    for act in ACTS:
        h, z = nan_like((M, N), BF16), nan_like((M, 2 * N), BF16)
        ops.linear_fwd(x, w, h, bias=bias, glu=act, z_out=z)
        dz = nan_like((M, 2 * N), BF16)
        ops.linear_dgrad(dy, w2, dz, glu_grad_of=z, glu=act)
        torch.cuda.synchronize()
        assert all(_same(z[r], zb) for r in (0, M - 1)), "z != bf16(bias)"
        h0, dv, dg = h[0].float(), dz[0, :N].float(), dz[0, N:].float()
        assert _same(h[M - 1], h[0]) and _same(dz[M - 1], dz[0])
        if act == "relu":
            a = torch.where(gt > 0, gt, torch.zeros_like(gt))
            assert _same(h0, (v * a).to(BF16)), "ReGLU h = bf16(zv relu(zg))"
            assert _same(dv, a.to(BF16)), "ReGLU dzv = bf16(1 a)"
            assert _same(dg, (torch.where(gt > 0, 1.0, 0.0) * v).to(BF16)), "ReGLU dzg = bf16([zg > 0] zv)"
            continue
        mod = (v.abs() <= 1e4) & (gt.abs() <= 1e4)           # no product leaves the fp32 range
        cols = torch.cat([mod, mod])
        check_h("edge GEGLU h (moderate z)", "gelu", h[:, mod], z[:, cols])
        ones = torch.ones(M, int(mod.sum()), dtype=F64, device=DEV)
        check_dz("edge GEGLU (moderate z)", "gelu", dz[:, cols], ones, ones, z[:, cols], 1)
        assert torch.isnan(h0[torch.isnan(v) | torch.isnan(gt) | (gt == float("-inf"))]).all()
        up = (gt == float("inf")) & torch.isfinite(v) & (v != 0)
        assert (h0[up] == v[up] * float("inf")).all()
        assert torch.isnan(dg[~torch.isfinite(gt)]).all()          # gelu' of a non-finite zg is NaN
    print(f"[{TAG}] edge values {edges} paired as (zv, zg): ReGLU bit for bit, GEGLU within its bounds")


def test_glu_entry_points_reject_bad_arguments(ops):
    from dalle_mtf_b200 import lib as L
    x = torch.zeros(128, 64, dtype=BF16, device=DEV)
    w = torch.zeros(64, 256, dtype=BF16, device=DEV)
    out = torch.empty(128, 128, dtype=BF16, device=DEV)
    z = torch.empty(128, 264, dtype=BF16, device=DEV)
    ops.linear_fwd(x, w, out, glu="relu", z_out=z[:, :256])                          # ldz = 264: fine
    with pytest.raises(L.DB200Error):                                                # ldz < 2N
        ops.gemm(x, w, out, 128, 128, 64, b_mn=True, glu="fwd", glu_act="relu", z=torch.empty(128, 128, dtype=BF16,
                                                                                              device=DEV))
    with pytest.raises(L.DB200Error):                                                # ldz % 8
        ops.linear_fwd(x, w, out, glu="gelu", z_out=torch.empty(128, 260, dtype=BF16, device=DEV)[:, :256])
    with pytest.raises(L.DB200Error):                                                # operand majors
        ops.gemm(x, w.T.contiguous(), out, 128, 128, 64, a_mn=False, b_mn=False, glu="fwd", glu_act="relu")
    with pytest.raises(L.DB200Error):                                                # ldb < 2N
        ops.gemm(x, w[:, :128].contiguous(), out, 128, 128, 64, b_mn=True, glu="fwd", glu_act="relu")
    with pytest.raises(L.DB200Error):                                                # N % 64
        ops.gemm(x, w, out, 128, 96, 64, b_mn=True, glu="fwd", glu_act="relu")
    with pytest.raises(L.DB200Error):
        ops.gemm(x, w, out, 128, 128, 64, b_mn=True, glu="fwd", glu_act="relu", residual=out)
    with pytest.raises(ValueError):
        ops.gemm(x, w, out, 128, 128, 64, b_mn=True, glu="fwd", glu_act="swish")
    with pytest.raises(L.DB200Error):
        ops.linear_fwd(x, w, out, glu="relu", relu=True)
    with pytest.raises(L.DB200Error):
        ops.linear_dgrad(out, w, x, glu_grad_of=z)                                     # no glu
    dz = torch.empty(128, 256, dtype=BF16, device=DEV)
    dy = torch.zeros(128, 64, dtype=BF16, device=DEV)
    w2 = torch.zeros(128, 64, dtype=BF16, device=DEV)
    zz = torch.zeros(128, 256, dtype=BF16, device=DEV)
    ops.linear_dgrad(dy, w2, dz, glu_grad_of=zz, glu="gelu")
    with pytest.raises(L.DB200Error):                                                # ldd < 2N
        ops.gemm(dy, w2, dz[:, :128], 128, 128, 64, mode=L.EPI_RELU_BWD, aux=zz, glu="bwd", glu_act="relu",
                 ldd=128)
    with pytest.raises(L.DB200Error):                                                # ldaux < 2N
        ops.gemm(dy, w2, dz, 128, 128, 64, mode=L.EPI_RELU_BWD, aux=zz[:, :128].contiguous(), glu="bwd",
                 glu_act="relu")
    lib = L.load()
    e = L.GemmEpilogue()
    e.mode, e.alpha = L.EPI_STORE, 1.0
    args = (None, L.ptr(x), 0, 64, L.ptr(w), 1, 256, L.ptr(out), 128, 128, 128, 64)
    assert lib.db200_gemm_bf16_glu(*args, None, 0, None, 0) != 0                     # NULL epilogue
    assert lib.db200_gemm_bf16_glu(*args, ctypes.byref(e), 2, None, 0) != 0          # act
    assert b"act" in lib.db200_last_error()
    assert lib.db200_gemm_bf16_glu(None, None, 0, 64, L.ptr(w), 1, 256, L.ptr(out), 128, 128, 128, 64,
                                   ctypes.byref(e), 0, None, 0) != 0                 # NULL A
    assert lib.db200_gemm_bf16_glu(None, L.ptr(x), 0, 64, L.ptr(w), 1, 256, None, 128, 128, 128, 64,
                                   ctypes.byref(e), 0, None, 0) != 0                 # NULL D
    e.mode = L.EPI_CE_GRAD
    assert lib.db200_gemm_bf16_glu_bwd(None, L.ptr(dy), 0, 64, L.ptr(w2), 0, 64, L.ptr(dz), 256, 128, 128, 64,
                                       ctypes.byref(e), 0) != 0                      # mode
    e.mode = L.EPI_RELU_BWD
    e.aux, e.ldaux = L.ptr(zz), 256
    assert lib.db200_gemm_bf16_glu_bwd(None, L.ptr(dy), 0, 64, L.ptr(w2), 0, 64, L.ptr(dz), 256, 128, 128, 64,
                                       ctypes.byref(e), 5) != 0                      # act
    e.aux = None
    assert lib.db200_gemm_bf16_glu_bwd(None, L.ptr(dy), 0, 64, L.ptr(w2), 0, 64, L.ptr(dz), 256, 128, 128, 64,
                                       ctypes.byref(e), 0) != 0                      # no aux
    torch.cuda.synchronize()


# ================================================================================================ engines vs oracle
def _params(cfg, seed):
    from oracle import dalle as O
    from oracle import dalle_glu as OGL
    p = OGL.init_params(O.init_params(cfg, seed), cfg, seed + 7)
    g = torch.Generator().manual_seed(seed + 1)
    d = cfg.n_embd
    for k in p:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            p[k] = torch.randn(p[k].shape, generator=g) * 0.02
        if k.endswith("/g"):
            p[k] = 1 + torch.randn(p[k].shape, generator=g) * 0.05
        if k.endswith("mlp_linear_1/kernel"):        # zg = LN2(x) W1 + b1 with std ~2: the curved part of GELU
            p[k] = p[k] * (100.0 / math.sqrt(d))
        if k.endswith("mlp_linear_1/bias"):
            p[k] = torch.randn(p[k].shape, generator=g) * 0.5
    return p


def _value_half(p, cfg, grads=False):
    """The ungated model inside a gated parameter (or gradient) dict: W1 / b1 cut to their value half."""
    out = dict(p)
    n = 4 * cfg.n_embd
    for l in range(cfg.n_layers):
        k, b = f"layer_{l}/mlp/mlp_linear_1/kernel", f"layer_{l}/mlp/mlp_linear_1/bias"
        out[k], out[b] = p[k][:, :n].contiguous(), p[b][:n].contiguous()
    return out


def engine_case(name, act, d, L, H, tv, iv, ts, isl, B, seed, recompute=False, attention_types=None, kernel=3,
                dropout=None, rotary=None, mutations=False):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    from oracle import dalle_glu as OGL
    layers = None
    if attention_types is not None:
        import conv_oracle as OC
        cfg = OC.ConvConfig(d, L, H, tv, iv, ts, isl, attention_types=tuple(attention_types),
                            local_attention_radius=8, conv_attention_kernel=kernel)
        layers = OC
    else:
        cfg = O.DalleConfig(d, L, H, tv, iv, ts, isl)
    spec = None if dropout is None else (dropout[0], dropout[1], 3, 0)
    params = _params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 2)
    tokens = O.assemble_tokens(torch.randint(0, tv - 1, (B, ts), generator=g),
                               torch.randint(0, iv, (B, isl), generator=g), tv)

    def oracle(mutate=None, gated=True, p=params):
        return [OGL.loss_and_grads(p, tokens, cfg, spec, bf16=bf, activation=act, gated=gated, mutate=mutate,
                                   layers=layers, rotary=rotary) for bf in (False, True)]

    o32, o16 = oracle()
    kw = dict(dropout=dropout[0], dropout_seed=dropout[1]) if dropout is not None else {}
    if rotary is not None:
        kw.update(rotary_dim=rotary[0], rotary_base=rotary[1])
    eng = DalleEngine(d, L, H, tv, iv, ts, isl, recompute_grad=recompute, attention_types=attention_types,
                      local_attention_radius=8, conv_attention_kernel=kernel, activation=act, gated_mlp=True, **kw)
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
        from dalle_mtf_b200 import ops as OPS
        lg = torch.empty(T, eng.Vpad, dtype=F32, device=DEV)
        eng.forward(tok, loss_accum=torch.zeros(1, device=DEV), step=3)
        OPS.gemm(eng._bufs["hf"], eng.W("wout"), lg, T, eng.Vpad, d, a_mn=False, b_mn=True, bias=eng.P("bout"))
        lg = lg.view(B, -1, eng.Vpad)[:, :, :eng.V].cpu()
    else:
        lg = eng.logits(tok).float().cpu()
    bad = GE._violations(loss, rows, lg, grads, o32, o16)
    zg = eng._bufs["layers"][0]["z1"][:, 4 * d:].float()
    print(f"[{TAG}] {name} {act}: loss {loss:.6f} oracle {o32[0].item():.6f}, logits relfro {relfro(lg, o32[2]):.2e} "
          f"(reference bf16 policy {relfro(o16[2], o32[2]):.2e}), zg std {zg.std().item():.2f}, violations {bad}")
    assert not bad, bad
    if mutations:
        for m in ("swap", "shift64"):
            vb = GE._violations(loss, rows, lg, grads, *oracle(m))
            print(f"[{TAG}] {name} {act} against the {m} mutant: {len(vb)} rules broken, e.g. {vb[:3]}")
            assert vb, f"{name}: the engine also matches the {m} mutant"
        half = _value_half(params, cfg)
        u32, u16 = oracle(gated=False, p=half)
        vb = GE._violations(loss, rows, lg, _value_half(grads, cfg), u32, u16)
        print(f"[{TAG}] {name} {act} against the ungated oracle: {len(vb)} rules broken, e.g. {vb[:3]}")
        assert vb, f"{name}: the engine also matches the ungated oracle"
    return eng


@pytest.mark.parametrize("act", ACTS)
def test_engine_matches_the_glu_oracle_and_not_the_mutants(act):
    engine_case("d256 L2", act, 256, 2, 2, 300, 64, 24, 40, 2, seed=21, mutations=True)


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("variant", [dict(dropout=((0.1, 0.1, 0.1), 7)), dict(recompute=True),
                                     dict(attention_types=["local", "axial_row", "conv", "global"], L=4),
                                     dict(rotary=(64, 10000.0))],
                         ids=["dropout", "recompute", "mixed", "rotary"])
def test_engine_variants_match_the_glu_oracle(act, variant):
    v = dict(variant)
    L = v.pop("L", 2)
    if v.get("attention_types"):
        engine_case(f"d256 L{L} {v['attention_types']}", act, 256, L, 2, 300, 64, 16, 64, 2, seed=22, **v)
    else:
        engine_case(f"d256 L{L} {variant}", act, 256, L, 2, 300, 64, 24, 40, 2, seed=22, **v)


def test_dalle_example_geometry_matches_the_geglu_oracle():
    engine_case("EX d512 L6 H4 S1280 V50771 B1", "gelu", 512, 6, 4, 50258, 512, 256, 1024, 1, seed=23)


# ================================================================================================ training steps
def _small(seed=0):
    from oracle import dalle as O
    cfg = O.DalleConfig(256, 2, 2, 300, 60, 40, 64)
    params = _params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    tokens = torch.cat([torch.randint(0, 300, (4, 40), generator=g), torch.randint(300, 360, (4, 64), generator=g)], 1)
    return cfg, params, tokens.to(I32).to(DEV)


@pytest.mark.parametrize("act", ACTS)
def test_two_gated_steps_are_bit_identical(act):
    g = torch.Generator().manual_seed(6)
    tok = torch.randint(0, 299, (4, 64), generator=g).to(I32).to(DEV)
    from dalle_mtf_b200.dalle_engine import DalleEngine
    outs = []
    for _ in range(2):
        eng = DalleEngine(256, 2, 2, 300, 64, 24, 40, activation=act, gated_mlp=True, dropout=(0.1, 0.1, 0.1),
                          dropout_seed=2)
        eng.init_params(3)
        assert eng.W("l0.w1").shape == (256, 2048)
        for step in range(2):
            eng.zero_grads()
            eng.forward(tok, step=step)
            eng.backward(1.0 / tok.numel())
            eng.optimizer_step(1e-3)
        torch.cuda.synchronize()
        outs.append((eng.grads.clone(), eng.master.clone(), eng.shadow.clone()))
    for a, b in zip(*outs):
        assert torch.equal(_bits(a), _bits(b))


def test_in_process_ranks_equal_one_rank_with_micro_batches_bitwise(monkeypatch, tmp_path):
    """tests/test_data_parallel_gpu.py's criterion (bit for bit), with the gated MLP and every feature."""
    from test_data_parallel_gpu import FEATURES, _Rec, _check_coverage, _dalle_data, _dalle_params, _dalle_ranks, \
        _dalle_reference, _seq_len, STEPS
    rec = _Rec(monkeypatch)
    for act, W in (("gelu", 2), ("relu", 3)):
        extra = dict(FEATURES, gated_mlp=True, activation_function=act)
        B = 12
        make = lambda **kw: _dalle_params(tmp_path, extra, train_batch_size=B, **kw)      # noqa: E731
        p = make()
        feats, caps = _dalle_data(p, B, seed=W)
        ref, n, aux_off = _dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * _seq_len(p)), feats, caps,
                                           W)
        group, chk, (n_r, aux_r) = _dalle_ranks(rec, make, feats, caps, W, ref)
        assert (n_r, aux_r) == (n, aux_off)
        _check_coverage(group.trace, n, aux_off, STEPS)
        chk.assert_clean()
        print(f"[{TAG}] {act} W={W}: {chk.bitwise} tensors bitwise equal to one rank with {W} micro-batches")


@pytest.mark.parametrize("act", ACTS)
def test_zero1_gated_step_equals_the_replicated_step_bitwise(act):
    from test_zero1_gpu import Loopback, _twin_from, assert_same_bits
    cfg, params, tok = _small(11)
    # bf16-representable values: ZeRO-1 keeps the vector parameters as fp32 copies of their bf16 values
    params = {k: v.to(BF16).float() for k, v in params.items()}
    kw = dict(gated_mlp=True, activation=act)
    grp = Loopback(2)
    grp.engines = ranks = [_engine(cfg, zero=grp.member(r), **kw) for r in range(2)]
    twin = _engine(cfg, **kw)
    for e in [twin] + ranks:
        e.load_params(params)
    n = twin.n_params_padded
    _twin_from(twin, twin.master[:n].clone(), ranks[0])
    g_ref = _step(twin, tok)
    for r, e in enumerate(ranks):
        assert_same_bits(_step(e, tok), g_ref, f"ZeRO-1 rank {r} gated gradients")
    twin.optimizer_step(1e-3)
    for e in ranks:
        e.optimizer_step(1e-3)
    for r, e in enumerate(ranks):
        assert_same_bits(e.shadow[:n], twin.shadow[:n], f"ZeRO-1 rank {r} parameters after the step")
    # the sharded initialiser draws the [d, 8d] W1 as the replicated one does
    a, b = _engine(cfg, **kw), _engine(cfg, zero=grp.member(0), **kw)
    a.init_params(4)
    b.init_params(4)
    assert_same_bits(b.shadow[:n], a.shadow[:n], "ZeRO-1 initialisation of a gated model")


# ================================================================================================ checkpoints
def _batch():
    g = torch.Generator().manual_seed(3)
    return torch.rand(4, 16, 16, 3, generator=g) * 2 - 1, torch.randint(0, 299, (4, 12), generator=g)


def test_model_fn_logs_saves_and_resumes_bit_exactly(tmp_path):
    import itertools
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.models import DALLE
    img, cap = _batch()
    G = {"gated_mlp": True, "activation_function": "gelu"}
    plain = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path))
    gated = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **G))
    d = 256
    assert gated.engine.gated_mlp and not plain.engine.gated_mlp
    assert gated.engine.n_params() - plain.engine.n_params() == 2 * (4 * d * d + 4 * d)
    gated.train_op(img, cap)
    st = gated.state_fn()
    assert tuple(st["layer_0/mlp/mlp_linear_1/kernel"].shape) == (d, 8 * d)
    assert tuple(st["layer_0/mlp/mlp_linear_1/bias"].shape) == (8 * d,)
    a = gated.train_op(img, cap).clone()
    sa = [t.clone() for t in (gated.engine.master, gated.engine.adam_m, gated.engine.adam_v)]
    resumed = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **G))
    resumed.load_fn(st)
    b = resumed.train_op(img, cap)
    assert torch.equal(a, b)
    for x, y in zip(sa, (resumed.engine.master, resumed.engine.adam_m, resumed.engine.adam_v)):
        assert torch.equal(x, y)

    class Log:
        lines = []

        def info(self, msg):
            self.lines.append(msg)
    log = Log()
    p = _tiny_params(tmp_path / "est", **G)
    p.update(model_path=None, iterations=1)
    Estimator(dalle_model_fn, p, logger=log).train(lambda params: itertools.repeat((img, cap)), max_steps=2)
    assert sum(ln.startswith("step ") for ln in log.lines) == 2, log.lines
    m = DALLE(256, text_vocab_size=300, image_vocab_size=60, text_seq_len=40, image_seq_len=88, n_layers=1, n_heads=2,
              mode="eval", params={"gated_mlp": True})
    assert m.engine.gated_mlp and m.engine.glu == "relu"
    g = torch.Generator().manual_seed(9)
    tokens = torch.cat([torch.randint(0, 300, (2, 40), generator=g), torch.randint(300, 360, (2, 88), generator=g)], 1)
    loss, loss_batch = m.forward({"tokens": tokens})
    assert math.isfinite(loss.item()) and loss_batch.shape == (2, 128)


def test_a_checkpoint_of_the_other_kind_is_refused_naming_the_variable():
    from dalle_mtf_b200 import lib as L
    from test_zero1_gpu import Loopback
    cfg, params, _ = _small(5)
    half = _value_half(params, cfg)
    for zero in (False, True):
        for gated, p in ((True, half), (False, params)):
            eng = _engine(cfg, gated_mlp=gated, zero=Loopback(2).member(0) if zero else None)
            with pytest.raises(L.DB200Error, match="w1"):
                eng.load_params(p)


# ================================================================================================ generation
def _gated_model(act, d=256, L=2, H=2, tv=300, iv=64, ts=24, isl=40, seed=3):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    cfg = O.DalleConfig(d, L, H, tv, iv, ts, isl)
    params = _params(cfg, seed)
    for k in params:
        if "wte" in k or "linear_out" in k:
            params[k] = params[k] * 4                       # sharper logits: clear arg-maxima
    eng = DalleEngine(d, L, H, tv, iv, ts, isl, activation=act, gated_mlp=True)
    eng.load_params(params)
    return eng


@pytest.mark.parametrize("act", ACTS)
def test_generation_greedy_graphed_prefill_and_guided(act):
    from dalle_mtf_b200.sampling import DalleSampler
    from test_prefill_gpu import greedy_agrees_with_full_forward
    eng = _gated_model(act)
    tv, ts, S = 300, 24, 64
    g = torch.Generator().manual_seed(9)
    text = torch.randint(0, tv, (3, ts), generator=g).to(I32).to(DEV)
    smp = DalleSampler(eng)
    toks, step_logits = smp.generate(text, temperature=0, return_logits=True)
    graphed = smp.generate_graphed(text, temperature=0)
    torch.cuda.synchronize()
    assert torch.equal(graphed, toks)
    greedy_agrees_with_full_forward(eng, toks, ts)
    full = eng.logits(toks)
    e = relfro(torch.stack(step_logits, 1), full[:, :S - 1])
    assert e < 2e-2, e
    for n in (1, 7):
        P = ts + n
        kc = [torch.zeros(3, eng.S, eng.H, eng.dh, dtype=BF16, device=DEV) for _ in range(eng.L)]
        vc = [torch.zeros_like(c) for c in kc]
        lg = eng.prefill(toks[:, :P].contiguous(), kc, vc)[:, :eng.V]
        ep = relfro(lg, step_logits[P - 1])
        print(f"[{TAG}] {act}: decode vs full {e:.2e}, prefill P={P} vs decoding {ep:.2e}")
        assert ep < 2e-2, ep
    torch.manual_seed(0)
    guided = smp.complete(text[:2], toks[:2, ts:ts + 8].contiguous() - eng.image_offset, samples_per_prompt=2,
                          guidance_scale=3.0, top_k=16)
    assert guided.shape == (4, S)
    assert ((guided[:, ts:] >= eng.image_offset) & (guided[:, ts:] < eng.image_offset + 64)).all()


def test_generate_cli_runs_on_a_tiny_gated_model(tmp_path):
    import json
    import numpy as np
    import generate_dalle
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.utils import save_checkpoint
    img, cap = _batch()
    p = _tiny_params(tmp_path, gated_mlp=True, activation_function="gelu")
    spec = dalle_model_fn(img, cap, "train", p)
    spec.train_op(img, cap)
    vae = spec.extra["vae"]
    save_checkpoint(str(tmp_path / "vae"), 1, {"vae/" + k: v for k, v in vae.export_params().items()})
    save_checkpoint(str(tmp_path / "dalle"), 1, spec.state_fn())
    vcfg = dict(p["vae_params"], model_path=str(tmp_path / "vae"))
    (tmp_path / "vae.json").write_text(json.dumps(vcfg))
    cfg = {k: v for k, v in p.items() if k != "vae_params"}
    cfg.update(vae_model=str(tmp_path / "vae.json"), model_path=str(tmp_path / "dalle"), predict_batch_size=2)
    (tmp_path / "gated.json").write_text(json.dumps(cfg))
    np.save(tmp_path / "ids.npy", np.array([[1, 2, 3] + [299] * 9, [4, 5] + [299] * 10], dtype=np.int64))
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "gated.json"), "--caption_ids", str(tmp_path / "ids.npy"),
                         "--out", str(out), "--temperature", "0"])
    toks = np.load(out / "tokens.npy")
    assert toks.shape == (2, spec.engine.S) and len(list(out.glob("*.png"))) == 2
    io = spec.engine.image_offset
    assert ((toks[:, 12:] >= io) & (toks[:, 12:] < io + 64)).all()


# ================================================================================================ launches
def test_gated_mlp_off_launches_what_it_launched_before(monkeypatch):
    """Without the key (absent or False) forward, backward and the optimiser step call the same ops in the same
    order with the same launch count; the gated model calls the same ops in the same order too."""
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops as O
    from oracle import dalle as OD
    cfg = OD.DalleConfig(256, 2, 2, 300, 60, 40, 64)
    params = OD.init_params(cfg, 10)
    g = torch.Generator().manual_seed(11)
    tok = torch.cat([torch.randint(0, 300, (4, 40), generator=g), torch.randint(300, 360, (4, 64), generator=g)],
                    1).to(I32).to(DEV)
    calls = []
    names = [n for n, f in vars(O).items() if callable(f) and not n.startswith("_") and getattr(f, "__module__", "")
             == O.__name__]
    for n in names:
        f = getattr(O, n)
        monkeypatch.setattr(O, n, (lambda n, f: lambda *a, **k: (calls.append(n), f(*a, **k))[1])(n, f))
    seqs, counts = [], []
    for kw in ({}, {"gated_mlp": False}, {"gated_mlp": True}):
        eng = _engine(cfg, **kw)
        eng.load_params(_params(cfg, 10) if kw.get("gated_mlp") else params)
        _step(eng, tok, 1.0 / tok.numel())
        calls.clear()
        n0 = L.launch_count()
        _step(eng, tok, 1.0 / tok.numel())
        eng.optimizer_step(1e-3)
        torch.cuda.synchronize()
        counts.append(L.launch_count() - n0)
        seqs.append(list(calls))
    assert seqs[0] == seqs[1] and counts[0] == counts[1]
    assert seqs[2] == seqs[0]
    print(f"[{TAG}] ops per step {len(seqs[0])}, launches {counts}")


def _glu_describe(base):
    """test_dalle_config_launches_gpu.describe with the GLU keywords of a gemm added to its class."""
    import launch_census as LC

    def describe(entry, A):
        d = base(entry, A)
        if d is None or entry != "gemm" or A.get("glu") is None:
            return d
        cls, info = d
        return LC.launch_class("gemm", **LC.fields(cls), glu=A["glu"], glu_act=A["glu_act"]), info
    return describe


def test_launch_census_of_a_gated_model_claims_every_glu_class(ops, monkeypatch):
    """dalle_example_b200 plus the key, recorded by test_dalle_config_launches_gpu.py's recorder (train, eval, eager
    and graphed decoding, prefill with guidance): every GLU launch class is launched again, at its recorded shape,
    by this module's kernel case, which checks it against float64; every other class is an ordinary product or a
    launch the ungated model makes."""
    import launch_census as LC
    import test_dalle_config_launches_gpu as CL
    import test_dalle_kernels_gpu as DK
    base = DK._config("dalle_example_b200")
    monkeypatch.setattr(CL, "describe", _glu_describe(CL.describe))
    for act in ACTS:
        monkeypatch.setattr(DK, "_config", lambda c, act=act: dict(base, gated_mlp=True, activation_function=act))
        classes = CL.record_config("dalle_example_b200")[0]
        glu = [c for c in classes if "glu" in LC.fields(c)]
        assert {LC.fields(c)["glu"] for c in glu} == {"fwd", "bwd"}, glu
        assert all(LC.fields(c)["glu_act"] == act for c in glu)
        assert not [c for c in classes if c[0] == "gemm" and LC.fields(c)["gelu"] is not None]
        shapes = sorted({(f["M"], f["K"], f["N"]) for f in map(LC.fields, glu)})   # (rows, d, 4d) both ways
        got = set()
        for M, d, N in shapes:
            got |= CL.replayed(lambda: glu_case(ops, f"census M={M}", M, d, N, act, seed=M + d))
        missing = [c for c in glu if c not in CL.claimed(glu, got, CL.OFFSETS)]
        print(f"[{TAG}] census {act}: {len(glu)} GLU classes at (M, d, 4d) {shapes}, unclaimed {missing}")
        assert not missing
