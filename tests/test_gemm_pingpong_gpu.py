"""Products with K <= 1024 and a STORE (no dropout), RELU_BWD or plain CE_GRAD epilogue run on the ping-pong GEMM
kernel: each consumer warpgroup owns a whole 128 x 128 tile and runs its epilogue from the accumulator registers.
Longer contractions, and the other epilogues, run on the kernel that hands the tile to an epilogue warpgroup through
shared memory.

Every case here runs a product twice: as it is, and with both operands zero-padded along K to 17 k-blocks, which takes
the other kernel.  Adding exact zeros leaves the accumulators as they were and both kernels add their k-blocks in the
same order, so STORE, RELU_BWD, CE_GRAD and the fused column sums must agree to the bit.  CE_STATS sums a row's
exponentials in column order and stays on the other kernel at every K, so that lse, and every gradient behind it, is
what it was; its twin must agree to the bit as well.  One float64 reference per epilogue guards against both kernels
being wrong together.

Shapes: ragged last tiles in M and N; K = 64 (one k-block per tile, the tightest schedule for the barriers that pass
the tensor cores between the warpgroups), 512 and 1024; one, two and three tiles per CTA, fewer tiles than SMs, and
the same under the SM reservations of test_reserved_sms_gpu.py; the products of the dalle_example step.
"""
import pytest
import torch

from float64_bounds import DEV, reserved_sms, sm_count

pytestmark = pytest.mark.gpu

K_OTHER = 17 * 64     # the first K past the ping-pong kernel's 16 k-blocks
BF16, F32 = torch.bfloat16, torch.float32


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def randn(shape, seed, scale=1.0, dtype=BF16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, device=DEV, generator=g) * scale).to(dtype)


def operands(M, N, K, a_mn, b_mn, seed, b_scale=None):
    """A and B as the kernel takes them, and their zero-padded twins with K_OTHER contraction rows."""
    A = randn((M, K), seed)
    B = randn((K, N), seed + 1, b_scale if b_scale is not None else K ** -0.5)
    Ap = torch.zeros(M, K_OTHER, dtype=BF16, device=DEV); Ap[:, :K] = A
    Bp = torch.zeros(K_OTHER, N, dtype=BF16, device=DEV); Bp[:K] = B
    lay_a = (lambda x: x.t().contiguous()) if a_mn else (lambda x: x)
    lay_b = (lambda x: x) if b_mn else (lambda x: x.t().contiguous())
    return A, B, (lay_a(A), lay_b(B)), (lay_a(Ap), lay_b(Bp))


def both(ops, M, N, K, short, padded, a_mn, b_mn, make_out, **kw):
    """The product on the ping-pong kernel and its zero-padded twin on the other one; returns the two outputs."""
    outs = []
    for (a, b), k in ((short, K), (padded, K_OTHER)):
        out = make_out()
        ops.gemm(a, b, out, M, N, k, a_mn=a_mn, b_mn=b_mn, **kw)
        outs.append(out)
    return outs


def relmax(got, ref):
    got, ref = got.double(), ref.double()
    assert torch.isfinite(got).all()
    return ((got - ref).abs().max() / (ref.abs().max() + 1e-30)).item()


def nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def same(a, b, what, finite=True):
    bad = ~torch.isfinite(a.float()) if finite else torch.isnan(a.float())
    assert not bad.any(), f"{what}: {bad.sum().item()} outputs not finite (never written over the NaN sentinel?)"
    assert torch.equal(a, b), f"{what}: {(a != b).sum().item()} of {a.numel()} elements differ between the kernels"


# ---------------------------------------------------------------------------------------------------- STORE
@pytest.mark.parametrize("K", [64, 512, 1024])
@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (False, False), (True, True), (True, False)])
def test_store_epilogues_on_a_ragged_shape(ops, K, a_mn, b_mn):
    M, N = 1096, 1160                       # 9 x 10 tiles, the last ones 72 rows / 8 columns wide
    A, B, short, padded = operands(M, N, K, a_mn, b_mn, seed=K)
    bias, res = randn((N,), 3, dtype=F32), randn((M, N), 4)
    prod = A.double() @ B.double()
    # bf16: bias + ReLU + residual
    kw = dict(bias=bias, relu=True, residual=res)
    o, o2 = both(ops, M, N, K, short, padded, a_mn, b_mn, lambda: nan((M, N), BF16), **kw)
    same(o, o2, "bf16 bias+relu+residual")
    assert relmax(o, torch.relu(prod + bias.double()) + res.double()) < 1e-2
    # bf16, nothing else
    o, o2 = both(ops, M, N, K, short, padded, a_mn, b_mn, lambda: nan((M, N), BF16))
    same(o, o2, "bf16 plain")
    assert relmax(o, prod) < 1e-2
    # fp32: alpha (a power of two: exact whether or not the compiler fuses it with the bias add) + bias
    o, o2 = both(ops, M, N, K, short, padded, a_mn, b_mn, lambda: nan((M, N), F32), alpha=0.5, bias=bias)
    same(o, o2, "fp32 alpha+bias")
    assert relmax(o, 0.5 * prod + bias.double()) < 1e-5
    # fp32 with a residual (the residual block and the output block share the staging buffer)
    o, o2 = both(ops, M, N, K, short, padded, a_mn, b_mn, lambda: nan((M, N), F32), residual=res)
    same(o, o2, "fp32 residual")
    assert relmax(o, prod + res.double()) < 1e-5


def test_store_into_a_wider_output(ops):
    """ldd > N: rows and columns outside the product keep what they held."""
    M, N, K, ldd = 200, 72, 512, 128
    A, B, short, padded = operands(M, N, K, False, True, seed=9)
    outs = []
    for (a, b), k in ((short, K), (padded, K_OTHER)):
        out = torch.full((M + 8, ldd), 7.0, dtype=BF16, device=DEV)
        ops.gemm(a, b, out, M, N, k, a_mn=False, b_mn=True)
        outs.append(out)
    same(outs[0], outs[1], "strided output")
    assert (outs[0][:, N:] == 7).all() and (outs[0][M:] == 7).all()
    assert relmax(outs[0][:M, :N], A.double() @ B.double()) < 1e-2


# ---------------------------------------------------------------------------------------------------- RELU_BWD
@pytest.mark.parametrize("K", [64, 512, 1024])
def test_relu_bwd_with_column_sums_on_a_ragged_shape(ops, K):
    from dalle_mtf_b200 import lib as L
    M, N = 1096, 1160
    A, B, short, padded = operands(M, N, K, False, False, seed=K + 1)
    H = randn((M, N), 6)
    cs = [torch.zeros(N, device=DEV), torch.zeros(N, device=DEV)]
    it = iter(cs)
    outs = []
    for (a, b), k in ((short, K), (padded, K_OTHER)):
        out = nan((M, N), BF16)
        ops.gemm(a, b, out, M, N, k, mode=L.EPI_RELU_BWD, aux=H, colsum=next(it))
        outs.append(out)
    same(outs[0], outs[1], "relu_bwd")
    same(cs[0], cs[1], "relu_bwd column sums")
    assert relmax(outs[0], (A.double() @ B.double()) * (H.double() > 0)) < 1e-2
    assert relmax(cs[0], outs[0].double().sum(0)) < 1e-5


# ---------------------------------------------------------------------------------------------------- cross-entropy
def cross_entropy_case(ops, T, K, V, Vpad, seed, with_bias=True, float64_bound=True):
    """CE_STATS -> ce_finish -> CE_GRAD with column sums, as they are and zero-padded along K."""
    from dalle_mtf_b200 import lib as L
    X, W, short, padded = operands(T, Vpad, K, False, True, seed, b_scale=2.0 * K ** -0.5)
    W[:, V:] = 0
    short[1][:, V:] = 0
    padded[1][:, V:] = 0
    g = torch.Generator(device=DEV).manual_seed(seed + 7)
    labels = torch.randint(0, V, (T,), device=DEV, generator=g, dtype=torch.int32)
    labels[:4] = torch.tensor([0, V - 1, 63, 64], dtype=torch.int32, device=DEV)
    bias = None
    if with_bias:
        bias = torch.zeros(Vpad, device=DEV)
        bias[:V] = randn((V,), seed + 8, 0.5, F32)
    nt = ops.ce_tiles(Vpad)
    alpha = 1.0 / T
    res = []
    for (a, b), k in ((short, K), (padded, K_OTHER)):
        pm, ps = nan((nt, T), F32), nan((nt, T), F32)
        ll, lse, lr, lsum = nan((T,), F32), nan((T,), F32), nan((T,), F32), torch.zeros(1, device=DEV)
        ops.gemm(a, b, None, T, Vpad, k, b_mn=True, mode=L.EPI_CE_STATS, bias=bias, labels=labels, part_max=pm,
                 part_sum=ps, label_logit=ll, n_valid=V)
        ops.ce_finish(pm, ps, ll, lse, lr, lsum)
        res.append(dict(pm=pm, ps=ps, ll=ll, lse=lse))
    for key, finite in (("ll", True), ("pm", False), ("ps", True), ("lse", True)):   # pm: -inf in all-padding half tiles
        same(res[0][key], res[1][key], f"CE_STATS {key}", finite=finite)
    if float64_bound:
        z = X.double() @ W.double()[:, :V]
        if with_bias:
            z = z + bias[:V].double()
        assert relmax(res[0]["lse"], torch.logsumexp(z, -1)) < 1e-4
    lse = res[0]["lse"]
    cs = [torch.zeros(Vpad, device=DEV), torch.zeros(Vpad, device=DEV)]
    dls = []
    for i, ((a, b), k) in enumerate(((short, K), (padded, K_OTHER))):
        dl = nan((T, Vpad), BF16)
        ops.gemm(a, b, dl, T, Vpad, k, b_mn=True, mode=L.EPI_CE_GRAD, alpha=alpha, bias=bias, labels=labels, lse=lse,
                 n_valid=V, colsum=cs[i])
        dls.append(dl)
    same(dls[0], dls[1], "dlogits")
    same(cs[0], cs[1], "dlogits column sums")
    assert (dls[0][:, V:] == 0).all()
    if float64_bound:
        p = torch.softmax(z, -1)
        p[torch.arange(T, device=DEV), labels.long()] -= 1
        assert relmax(dls[0][:, :V], p * alpha) < 1e-2
        assert relmax(cs[0], dls[0].double().sum(0)) < 1e-4


@pytest.mark.parametrize("K", [64, 512, 1024])
@pytest.mark.parametrize("V,Vpad", [(2000, 2048), (2000, 2184), (1990, 1992)])
def test_cross_entropy_epilogues(ops, K, V, Vpad):
    """Vpad 2184: the last two tiles, one of them 8 columns wide, lie wholly in the padding (their partials must be
    (-inf, 0) and their dlogits exact zeros); 1992: the valid columns end two columns before
    the padded width, inside a column pair's 8-column group.  T = 1101 ends inside a tile."""
    cross_entropy_case(ops, 1101, K, V, Vpad, seed=K + V)


def test_cross_entropy_without_bias(ops):
    cross_entropy_case(ops, 520, 512, 1000, 1024, seed=2, with_bias=False)


# ---------------------------------------------------------------------------------------------------- schedules
def store_twin_case(ops, M, N, K, what):
    A, B, short, padded = operands(M, N, K, False, True, seed=M + N + K)
    bias = randn((N,), 5, dtype=F32)
    o, o2 = both(ops, M, N, K, short, padded, False, True, lambda: nan((M, N), BF16), bias=bias)
    same(o, o2, what)
    assert relmax(o, A.double() @ B.double() + bias.double()) < 1e-2


@pytest.mark.parametrize("K", [64, 512])
@pytest.mark.parametrize("tiles_per_cta", [1, 2, 3, 5])
def test_tiles_per_cta(ops, K, tiles_per_cta):
    """A persistent grid of one CTA per SM walking exactly 1, 2, 3 or 5 tiles each: with one, the second warpgroup has
    no tile at all; with an odd number the first gets one more than the second."""
    sms = sm_count()
    store_twin_case(ops, 128 * sms - 5, 128 * tiles_per_cta, K, f"{tiles_per_cta} tiles per CTA")


@pytest.mark.parametrize("M,N", [(100, 64), (300, 200), (128 * 7, 128 * 9 + 8)])
def test_fewer_tiles_than_sms(ops, M, N):
    store_twin_case(ops, M, N, 64, "fewer tiles than SMs")
    store_twin_case(ops, M, N, 1024, "fewer tiles than SMs")


@pytest.mark.parametrize("k", [16, 4, 5])
def test_under_reserved_sms(ops, k):
    """The grids of test_reserved_sms_gpu.py: the persistent grid is min(tiles, SMs - k), so the tile lists of the
    CTAs, and with them the split between the two warpgroups, change; 5 leaves an odd grid."""
    with reserved_sms(k) as sm:
        store_twin_case(ops, 128 * sm + 40, 384, 64, f"reserved {k}")       # 3 tiles per CTA and three more
        store_twin_case(ops, 128 * (sm + 1), 128, 512, f"reserved {k}")     # one CTA walks two tiles
        cross_entropy_case(ops, 128 * sm - 3, 64, 250, 256, seed=k, float64_bound=False)


# ---------------------------------------------------------------------------------------------------- engine shapes
def test_dalle_example_products_match_the_other_kernel(ops):
    """The K = 512 products of the dalle_example step (d = 512, 32 sequences of 1280 tokens) with their operand majors
    and epilogues: q|k|v, the W1 forward, the two residual projections, the ReLU-masked dgrad with its bias gradient
    and a plain dgrad.  Bitwise equal to the zero-padded twin."""
    from dalle_mtf_b200 import lib as L
    T, d = 40960, 512
    for N, kw, b_mn in ((1536, dict(bias=True), True), (2048, dict(bias=True, relu=True), True),
                        (512, dict(bias=True, residual=True), True), (512, dict(), False)):
        A, B, short, padded = operands(T, N, d, False, b_mn, seed=N)
        args = {}
        if kw.get("bias"):
            args["bias"] = randn((N,), 11, dtype=F32)
        if kw.get("relu"):
            args["relu"] = True
        if kw.get("residual"):
            args["residual"] = randn((T, N), 12)
        o, o2 = both(ops, T, N, d, short, padded, False, b_mn, lambda: nan((T, N), BF16), **args)
        same(o, o2, f"STORE N={N} {sorted(kw)}")
        del A, B, short, padded, o, o2, args
    N = 2048
    A, B, short, padded = operands(T, N, d, False, False, seed=77)
    H = randn((T, N), 13)
    outs, cs = [], [torch.zeros(N, device=DEV), torch.zeros(N, device=DEV)]
    for i, ((a, b), k) in enumerate(((short, d), (padded, K_OTHER))):
        out = nan((T, N), BF16)
        ops.gemm(a, b, out, T, N, k, mode=L.EPI_RELU_BWD, aux=H, colsum=cs[i])
        outs.append(out)
    same(outs[0], outs[1], "RELU_BWD")
    same(cs[0], cs[1], "RELU_BWD column sums")


def test_vocabulary_products_match_the_other_kernel(ops):
    """CE_STATS (one kernel at every K) and CE_GRAD at the dalle_example vocabulary (50 771 ids padded to 50 816 columns, d = 512), two
    sequences of rows."""
    cross_entropy_case(ops, 2560, 512, 50771, 50816, seed=31, float64_bound=False)
