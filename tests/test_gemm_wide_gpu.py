"""Products with K > 1024, a STORE (no dropout) or RELU_BWD epilogue and at least two 128 x 256 tiles per SM run on
the wide GEMM kernel: two warpgroups of wgmma m64n256 on a 128 x 256 tile, the epilogue from the
accumulator registers.  Fewer tiles take the kernel with 128 x 128 tiles and an epilogue warpgroup.

Every case runs a product twice: whole, and in slices small enough to fall under the tile rule, which puts each slice
on the 128 x 128 kernel.  Both kernels give an element the same k16 MMA steps in the same k-block order and the same
epilogue expression, so outputs and fused column sums must agree to the bit; that also establishes that m64n256
accumulates an element exactly as m64n128 does.  Products with column sums are sliced by columns only: a column's sum
over the 32-row blocks is then added in the same order.  A profiled launch checks which kernel each side ran on, and
one float64 reference per epilogue guards against both being wrong together.

Shapes: ragged last tiles in M (one with rows for both warpgroups, one for the first only) and N (one whose second
128-column half is partly, one wholly past N); all four operand majors; an output inside a wider buffer; the long-K
products of the dalle_example and dalle_coco steps at their sizes; SMs reserved as in test_reserved_sms_gpu.py.  The
single-split ATOMIC vocabulary wgrad stays on the 128 x 128 kernel.
"""
import re

import pytest
import torch

from float64_bounds import DEV, reserved_sms, sm_count

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32
WIDE_MIN_TILES = 2   # 128 x 256 tiles per SM from which a product goes to the wide kernel (gemm.cu)


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def randn(shape, seed, scale=1.0, dtype=BF16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, device=DEV, generator=g) * scale).to(dtype)


def nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def operands(M, N, K, a_mn, b_mn, seed):
    """A [M, K] and B [K, N], and the tensors the kernel takes for the given majors."""
    A, B = randn((M, K), seed), randn((K, N), seed + 1, K ** -0.5)
    return A, B, (A.t().contiguous() if a_mn else A), (B if b_mn else B.t().contiguous())


def gemm_kernels(fn):
    """Names of the GEMM kernels fn launches (its column-sum and split-K reductions aside)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {m.group(0) for e in prof.events() if e.device_type == DeviceType.CUDA
            for m in [re.search(r"gemm_(tc|pp|wide)_kernel", e.name)] if m}


def slices(M, N):
    """Rows and columns of the slices that stay under the wide kernel's tile rule: all rows and the widest multiple
    of 256 columns that fits, unless the rows alone make too many tiles."""
    limit = WIDE_MIN_TILES * sm_count()
    rows = M if -(-M // 128) < limit else 128 * (limit - 1)
    return rows, 256 * max(1, (limit - 1) // -(-rows // 128))


def both(ops, a, b, M, N, K, a_mn, b_mn, make_out, colsum=False, **kw):
    """The product whole (wide kernel) and in slices (128 x 128 kernel): two (output, column sums) pairs.  make_out()
    gives a fresh output, possibly a view of a wider buffer; bias, residual, aux and the column sums are sliced with
    it."""
    res = []
    for sliced in (False, True):
        out = make_out()
        cs = torch.zeros(N, device=DEV) if colsum else None

        def run():
            R, W = slices(M, N) if sliced else (M, N)
            assert cs is None or R == M, "column sums need whole columns"
            for m0 in range(0, M, R):
                m1 = min(M, m0 + R)
                for n0 in range(0, N, W):
                    n1 = min(N, n0 + W)
                    sub = {k: (v[n0:n1] if k == "bias" else v[m0:m1, n0:n1] if k in ("residual", "aux") else v)
                           for k, v in kw.items()}
                    if cs is not None:
                        sub["colsum"] = cs[n0:n1]
                    ops.gemm(a[:, m0:m1] if a_mn else a[m0:m1], b[:, n0:n1] if b_mn else b[n0:n1], out[m0:m1, n0:n1],
                             m1 - m0, n1 - n0, K, a_mn=a_mn, b_mn=b_mn, **sub)

        got = gemm_kernels(run)
        want = "gemm_tc_kernel" if sliced else "gemm_wide_kernel"
        assert got == {want}, f"{'sliced' if sliced else 'whole'} {M}x{N}x{K}: ran {sorted(got)}, expected {want}"
        res.append((out, cs))
    return res


def same(a, b, what):
    bad = ~torch.isfinite(a.float())
    assert not bad.any(), f"{what}: {bad.sum().item()} outputs not finite (never written over the NaN sentinel?)"
    assert torch.equal(a, b), f"{what}: {(a != b).sum().item()} of {a.numel()} elements differ between the kernels"


def relmax(got, ref):
    got, ref = got.double(), ref.double()
    assert torch.isfinite(got).all()
    return ((got - ref).abs().max() / (ref.abs().max() + 1e-30)).item()


def ragged_m(n_wide, rows_in_last):
    """M with at least WIDE_MIN_TILES 128 x 256 tiles per SM and `rows_in_last` rows in the last 128-row tile."""
    return 128 * -(-WIDE_MIN_TILES * sm_count() // n_wide) + rows_in_last


# ---------------------------------------------------------------------------------------------------- STORE
@pytest.mark.parametrize("N,rows_in_last", [(1160, 72), (1032, 40)])
@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (False, False), (True, True), (True, False)])
def test_store_epilogues_on_a_ragged_shape(ops, N, rows_in_last, a_mn, b_mn):
    """N = 1160: the last 256-wide tile holds 136 columns; 1032: 8, so its second half lies wholly past N.
    72 rows in the last tile reach the second warpgroup, 40 do not."""
    K = 1088
    M = ragged_m(-(-N // 256), rows_in_last)
    A, B, a, b = operands(M, N, K, a_mn, b_mn, seed=N + rows_in_last)
    bias, res = randn((N,), 3, dtype=F32), randn((M, N), 4)
    (o, _), (o2, _) = both(ops, a, b, M, N, K, a_mn, b_mn, lambda: nan((M, N), BF16), bias=bias, relu=True,
                           residual=res)
    same(o, o2, "bf16 bias+relu+residual")
    assert relmax(o, torch.relu(A.double() @ B.double() + bias.double()) + res.double()) < 1e-2
    (o, _), (o2, _) = both(ops, a, b, M, N, K, a_mn, b_mn, lambda: nan((M, N), BF16))
    same(o, o2, "bf16 plain")
    # fp32: alpha (a power of two: exact whether or not the compiler fuses it with the bias add) + bias
    (o, _), (o2, _) = both(ops, a, b, M, N, K, a_mn, b_mn, lambda: nan((M, N), F32), alpha=0.5, bias=bias)
    same(o, o2, "fp32 alpha+bias")
    (o, _), (o2, _) = both(ops, a, b, M, N, K, a_mn, b_mn, lambda: nan((M, N), F32), residual=res)
    same(o, o2, "fp32 residual")


def test_store_into_a_wider_output(ops):
    """ldd > N: columns outside the product keep what they held."""
    N, K, ldd = 1032, 2048, 1160
    M = ragged_m(5, 72)
    A, B, a, b = operands(M, N, K, False, True, seed=9)
    outs = both(ops, a, b, M, N, K, False, True, lambda: torch.full((M, ldd), 7.0, dtype=BF16, device=DEV)[:, :N])
    (o, _), (o2, _) = outs
    same(o, o2, "strided output")
    assert (o.as_strided((M, ldd - N), (ldd, 1), N) == 7).all()


# ---------------------------------------------------------------------------------------------------- RELU_BWD
@pytest.mark.parametrize("N,rows_in_last", [(1160, 72), (1032, 40)])
def test_relu_bwd_with_column_sums_on_a_ragged_shape(ops, N, rows_in_last):
    from dalle_mtf_b200 import lib as L
    K = 1088
    M = ragged_m(-(-N // 256), rows_in_last)
    A, B, a, b = operands(M, N, K, False, False, seed=N + 1)
    H = randn((M, N), 6)
    (o, cs), (o2, cs2) = both(ops, a, b, M, N, K, False, False, lambda: nan((M, N), BF16), mode=L.EPI_RELU_BWD,
                              aux=H, colsum=True)
    same(o, o2, "relu_bwd")
    same(cs, cs2, "relu_bwd column sums")
    assert relmax(o, (A.double() @ B.double()) * (H.double() > 0)) < 1e-2
    assert relmax(cs, o.double().sum(0)) < 1e-4


# ---------------------------------------------------------------------------------------------------- engine shapes
def engine_products(ops, T, d, Vpad, seed):
    """The long-K products of one training step with T token rows, width d and padded vocabulary Vpad: the
    vocabulary dgrad, the second MLP product (bias + residual), the first one's dgrad and the q|k|v dgrad."""
    cases = ((T, d, Vpad, False, False, dict()),
             (T, d, 4 * d, False, True, dict(bias=True, residual=True)),
             (T, d, 4 * d, False, False, dict()),
             (T, d, 3 * d, False, False, dict()))
    for i, (M, N, K, a_mn, b_mn, kw) in enumerate(cases):
        g = torch.Generator(device=DEV).manual_seed(seed + i)
        a = torch.randn((K, M) if a_mn else (M, K), device=DEV, generator=g).to(BF16)
        b = (torch.randn((K, N) if b_mn else (N, K), device=DEV, generator=g) * K ** -0.5).to(BF16)
        args = dict(kw)
        if args.pop("bias", False):
            args["bias"] = randn((N,), seed + 11, dtype=F32)
        if args.pop("residual", False):
            args["residual"] = randn((M, N), seed + 12)
        (o, _), (o2, _) = both(ops, a, b, M, N, K, a_mn, b_mn, lambda: nan((M, N), BF16), **args)
        same(o, o2, f"{M}x{N}x{K} {sorted(kw)}")
        del a, b, args, o, o2
        torch.cuda.empty_cache()


def test_dalle_example_products(ops):
    """32 sequences of 1280 tokens, d = 512, 50 771 ids padded to 50 816 columns."""
    engine_products(ops, 40960, 512, 50816, seed=41)


def test_dalle_coco_products(ops):
    """16 sequences of 1280 tokens, d = 1024, 58 451 ids padded to 58 496 columns."""
    engine_products(ops, 20480, 1024, 58496, seed=43)


# ---------------------------------------------------------------------------------------------------- schedules
@pytest.mark.parametrize("k", [16, 4, 5])
def test_under_reserved_sms(ops, k):
    """The grids of test_reserved_sms_gpu.py: the persistent grid is min(tiles, SMs - k) and the tile rule reads the
    reduced SM count; 5 leaves an odd grid."""
    from dalle_mtf_b200 import lib as L
    with reserved_sms(k):
        N, K = 1160, 1088
        M = ragged_m(5, 72)
        A, B, a, b = operands(M, N, K, False, True, seed=k)
        bias = randn((N,), 5, dtype=F32)
        (o, _), (o2, _) = both(ops, a, b, M, N, K, False, True, lambda: nan((M, N), BF16), bias=bias)
        same(o, o2, f"reserved {k}: STORE")
        H = randn((M, N), 6)
        (o, cs), (o2, cs2) = both(ops, a, b.t().contiguous(), M, N, K, False, False, lambda: nan((M, N), BF16),
                                  mode=L.EPI_RELU_BWD, aux=H, colsum=True)
        same(o, o2, f"reserved {k}: RELU_BWD")
        same(cs, cs2, f"reserved {k}: RELU_BWD column sums")


def test_vocabulary_wgrad_stays_on_the_128_wide_kernel(ops):
    """The single-split ATOMIC wgrad measured no faster on 128 x 256 tiles."""
    from dalle_mtf_b200 import lib as L
    A, B, a, b = operands(512, 50816, 1088, True, True, seed=5)
    D = torch.zeros(512, 50816, device=DEV)
    assert gemm_kernels(lambda: ops.gemm(a, b, D, 512, 50816, 1088, a_mn=True, b_mn=True,
                                         mode=L.EPI_ATOMIC)) == {"gemm_tc_kernel"}
