"""The kernels at the limits include/dalle_b200.h promises: sizes and offsets past 2^31 and 2^32 elements, dropout
counters whose high word hi32(n) is not 0, and the widest rows of the samplers.

Bounds and harnesses are those of test_dalle_kernels_gpu.py (float64 references, its module docstring), of
test_loss_weights_gpu.py (weighted cross-entropy) and of test_sampling_filter_gpu.py / test_guidance_gpu.py (kept sets
and draws); only the operand sizes and the dropout row0 are new here.  Outputs start as NaN.  Every case prints
`[abi-limits] <case>: worst err/bound r` (r = 0: bit for bit) and needs r < 1.  Large outputs sit inside a larger
allocation with GUARD sentinel elements on either side that must come back untouched.  A case whose device-memory
budget (from its buffer sizes, plus 4 GiB) is not free is skipped with a line that names the memory it needed.

A. Past 2^31 and 2^32 elements, dalle_example width (d = 512, V = 50 771, Vpad = 50 816).  Index arithmetic read
   before the first run, 64-bit on every path below:
   - GEMM (gemm.cu, gemm_common.cuh): TMA maps take uint64 dims and byte strides; stage_flush / stage_fetch_bf16 form
     (long long)row * ld + col and step rows by ld * 4 * esz in long long; the f32 STORE and ATOMIC epilogues write
     D + (long long)row * ldd; the split-K slice base is (long long)split * M * ldd and reduce_splits_add_kernel reads
     ws[k * mn + i] with mn and i long long; CE_STATS partials sit at (long long)tile * M + row, colsum partials at
     (long long)(row0 >> 5) * N; the dropout block index is dropout_elem_block's (row0 + r) * cols + c in long long.
   - ce_finish / ce_finish_weighted (rowops.cu): partials read at (long long)tile * M + row; rows and tiles are int.
   - cast_f32_bf16 / cast_bf16_f32 / split_f32 / sqnorm / adam (rowops.cu, optim.cu): size_t n, size_t grid-stride
     index, vector index i and tail (nv << 3 or nv << 2) + threadIdx.x in size_t; the grid is capped at 8-16 x SM.
   - crop_resize_kernel (data_ops.cu): image base packed + offsets[b] with int64 offsets, pixel offsets in long long.
   Vocabulary chain at T = 43 520 (34 sequences: T Vpad > 2^31) and T = 85 760 (67 sequences: > 2^32): CE_STATS ->
   ce_finish -> CE_GRAD with the fused colsum, then the dgrad dl W^T (K = Vpad) and the split-K wgrad x^T dl (K = T)
   that read that gradient, then the weighted CE_GRAD with z-loss into the same buffer.  Every row slab (DK.SLAB) is
   compared, so the rows either side of element 2^31 (and 2^32) are too.  The fp32 STORE of logits() at T = 43 520.
   Flat kernels at n = 2^31 + 37: each input slab of FLAT elements is drawn from (seed, slab index), so the float64
   check regenerates it; slab 0, the slab below 2^31 and the tail slab are compared.  image_crop_resize_normalize
   reads one image at an odd byte offset above 2^32 of a 4.3 GB buffer, bit for bit against oracle/data.py, next to a
   different image at that offset minus 2^32.
B. Dropout counters with hi32(n) != 0: elementwise cols = 512 from row0 = 2^25 - 3 (n crosses 2^32 at local row 3);
   attention H = 32, S = 1280 from sequence 327 (inside head 21); caption dropout from sequence 2^34 - 5.  The masks
   equal oracle/philox.py (whose high word test_abi_limits_cpu.py checks against a Python-int Philox), and every
   kernel that regenerates a mask matches float64 given the mask.
C. Sampler rows of 32 769, 50 771 and 51 200 ids (the filtered kernels' one-CTA limit), 51 201 rejected before any
   launch, and the unfiltered sampler at 58 496 ids.

On an H100 80GB HBM3 (700 W power limit) the module takes 59 s of wall time including start-up (52 s from the first
case on), and its peak device memory is 38.3 GiB (the Adam case: p, m, v, g and the bf16 shadow at n = 2^31 + 37); the
vocabulary chain peaks at 12.1 GiB (T = 43 520) and 16.2 GiB (T = 85 760), the casts at 16.3 GiB, logits() at 12.8 GiB.
"""
import functools
import math
import time
import types

import numpy as np
import pytest
import torch

import float64_bounds
import test_dalle_kernels_gpu as DK
import test_guidance_gpu as GU
import test_loss_weights_gpu as LW
import test_sampling_filter_gpu as SF
from float64_bounds import DEV, U

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
TAG = "abi-limits"
GIB = 2.0 ** 30
GUARD = 1 << 16                      # sentinel elements on either side of a large output
CONFIG = "dalle_example_b200"
VOCAB_T = {43520: 2 ** 31, 85760: 2 ** 32}   # tokens per GPU -> the element boundary its dlogits crosses
N_FLAT = 2 ** 31 + 37
FLAT = 1 << 24                       # elements per generated / compared slab of a flat buffer
ELEM_ROW0, ELEM_ROWS, ELEM_COLS = 2 ** 25 - 3, 8, 512
ATTN_ROW0, ATTN_B, ATTN_H, ATTN_S, ATTN_DH = 327, 2, 32, 1280, 128
CAP_ROW0, CAP_B = 2 ** 34 - 5, 10

_PEAK = [0]


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    t0 = time.time()
    yield _ops
    print(f"[{TAG}] module wall time {time.time() - t0:.0f} s, peak device memory {_PEAK[0] / GIB:.1f} GiB")


@pytest.fixture(autouse=True)
def _case(request, monkeypatch):
    """Case lines of the reused harnesses carry this module's tag; every case starts and ends with the cache freed."""
    tagged = functools.partial(float64_bounds.check, tag=TAG)
    monkeypatch.setattr(DK, "TAG", TAG)
    monkeypatch.setattr(DK, "check", tagged)
    monkeypatch.setattr(LW, "check", tagged)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated()
    _PEAK[0] = max(_PEAK[0], peak)
    print(f"[{TAG}] {request.node.name}: peak device memory {peak / GIB:.1f} GiB")
    torch.cuda.empty_cache()


def need(gib, what):
    """Skip (with a printed reason) unless the device has gib + 4 GiB free: the machines are shared."""
    free, _ = torch.cuda.mem_get_info()
    if free < (gib + 4) * GIB:
        msg = f"[{TAG}] {what}: skipped, needs {gib:.1f} + 4 GiB of device memory, {free / GIB:.1f} GiB free"
        print(msg)
        pytest.skip(msg)


def guarded(shape, dtype, fill=math.nan):
    """A `shape` output (filled with `fill`, or left for the caller when None) inside a buffer with GUARD random
    sentinel elements on either side."""
    n = math.prod(shape)
    buf = torch.empty(n + 2 * GUARD, dtype=dtype, device=DEV)
    sent = (torch.rand(2 * GUARD, generator=DK._gen(n % 100003), device=DEV) * 1000 + 1).to(dtype)
    buf[:GUARD], buf[-GUARD:] = sent[:GUARD], sent[GUARD:]
    out = buf[GUARD:GUARD + n].view(shape)
    if fill is not None:
        out.fill_(fill)
    return types.SimpleNamespace(buf=buf, out=out, sent=sent)


def assert_untouched(name, gd):
    assert torch.equal(gd.buf[:GUARD], gd.sent[:GUARD]), f"{name}: a write landed before the output"
    assert torch.equal(gd.buf[-GUARD:], gd.sent[GUARD:]), f"{name}: a write landed past the output"


def exact(name, got, want):
    """got equals want bit for bit (same dtype); prints the case line with r = 0."""
    assert got.dtype == want.dtype and got.shape == want.shape
    iv = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[got.element_size()]
    same = torch.equal(got.view(iv), want.view(iv))
    print(f"{float64_bounds.prefix()}[{TAG}] {name}: worst err/bound {0.0 if same else math.inf:.4f} (bit for bit)")
    assert same, f"{name}: not bit for bit"


# ------------------------------------------------------------------------------------------------------- A: vocabulary
def run_product(ops, name, a, b, M, N, K, *, a_mn, b_mn, mode, out_dtype=BF16, bias=None, seed=0):
    """One product on existing operands through DK.run_gemm / DK.check_gemm, into a guarded output (ATOMIC: onto a
    random base); split_k = 0 (the engine's wgrad rule) for ATOMIC."""
    from dalle_mtf_b200 import lib as L
    atomic = mode == L.EPI_ATOMIC
    o = types.SimpleNamespace(M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, mode=mode, relu=False, split_k=0 if atomic else 1,
                              dropout=None, a=a, b=b, bias=bias, res=None, aux=None, cs_base=None, colsum=None,
                              keep=None, base=None)
    gd = guarded((M, N), F32 if atomic else out_dtype, fill=None if atomic else math.nan)
    if atomic:
        o.base = DK._randn(M, N, g=DK._gen(seed))
        gd.out.copy_(o.base)
    o.out = gd.out
    DK.run_gemm(ops, o)
    splits = DK.gemm_splits(M, N, K, mode, o.split_k, DK._sm())
    r = DK.check_gemm(f"{name} {DK._mode_name(mode)} {M}x{N}x{K} splits={splits}", o, splits)
    assert_untouched(name, gd)
    return r


def _vocab_operands(ops, T):
    K, V, Vpad, h, W, bias, labels = DK.real_vocabulary_operands(ops, CONFIG, T)
    assert (K, V, Vpad) == (512, 50771, 50816)
    return K, V, Vpad, h, W, bias, labels


@pytest.mark.parametrize("T", list(VOCAB_T))
def test_vocabulary_chain_past_the_32_bit_element_boundary(ops, T):
    from dalle_mtf_b200 import lib as L
    Vpad, boundary = 50816, VOCAB_T[T]
    dl_gib = T * Vpad * 2 / GIB
    need(dl_gib + 5.0, f"vocabulary chain T={T} ({dl_gib:.1f} GiB of dlogits + 5 GiB of float64 slabs)")
    K, V, Vpad, h, W, bias, labels = _vocab_operands(ops, T)
    row = boundary // Vpad                          # the row holding element `boundary` of dlogits
    assert boundary < T * Vpad and 0 < row < T - 1
    print(f"[{TAG}] T={T}: dlogits has {T * Vpad} elements, element {boundary} in row {row}")
    gd = guarded((T, Vpad), BF16)
    tag = f"T={T} Vpad={Vpad}"
    DK.run_cross_entropy(ops, f"{tag} CE", T, K, V, Vpad, labels=labels, h=h, W=W, bias=bias, dl=gd.out)
    assert_untouched(f"{tag} dlogits", gd)
    dl = gd.out
    # the products of the engine's backward that read dlogits: dx = dl wout^T (wout stored [K][Vpad]) and
    # dwout += x^T dl (x stored [T][K], dl [T][Vpad]: both mn-major), split-K over T
    run_product(ops, f"{tag} dgrad", dl, W, T, K, Vpad, a_mn=False, b_mn=False, mode=L.EPI_STORE)
    run_product(ops, f"{tag} wgrad", h, dl, K, Vpad, T, a_mn=True, b_mn=True, mode=L.EPI_ATOMIC, seed=T)
    dl.fill_(math.nan)
    cfg = DK._config(CONFIG)
    LW.run_weighted_ce(ops, f"{tag} weighted CE w=(1, 7) z=1e-4", T, K, V, Vpad, 1280, cfg["text_seq_len"],
                       labels=labels, h=h, W=W, bias=bias, weights=(1.0, 7.0), z=1e-4, global_batch=T // 1280, dl=dl)
    assert_untouched(f"{tag} weighted dlogits", gd)


def test_logits_fp32_store_past_2_31_elements(ops):
    """logits() writes fp32 [T, Vpad] logits through the STORE epilogue with the bias (the one fp32 STORE the engine
    records); at T = 43 520 that is 2.2e9 elements (8.2 GiB)."""
    from dalle_mtf_b200 import lib as L
    T, Vpad = 43520, 50816
    need(T * Vpad * 4 / GIB + 3.0, f"logits() fp32 STORE T={T} ({T * Vpad * 4 / GIB:.1f} GiB of logits + 3 GiB)")
    calls = DK.engine_calls(ops, CONFIG)[0]
    f32 = [c for c in calls if c[0] == "gemm" and c[6] == L.EPI_STORE and c[7] == "torch.float32"]
    assert len(f32) == 1 and f32[0][2:6] == (Vpad, 512, False, True) and f32[0][8], f32
    K, V, Vpad, h, W, bias, _ = _vocab_operands(ops, T)
    assert T * Vpad > 2 ** 31
    run_product(ops, f"logits() T={T}", h, W, T, Vpad, K, a_mn=False, b_mn=True, mode=L.EPI_STORE, out_dtype=F32,
                bias=bias)


# ------------------------------------------------------------------------------------------------------- A: flat buffers
def flat_slabs(n):
    return [(i, a, min(n, a + FLAT)) for i, a in enumerate(range(0, n, FLAT))]


def checked_slabs(n):
    """Slab 0, the slab that ends at element 2^31 and the tail slab (the vector kernels' scalar tail lies in it)."""
    s = flat_slabs(n)
    picked = [s[0], s[(2 ** 31) // FLAT - 1], s[-1]]
    assert picked[1][2] == 2 ** 31 and picked[2][1] == 2 ** 31 and picked[2][2] == n
    return picked


def adam_inputs(seed, i, length):
    """(p, g, m, v) of slab i, the magnitudes of test_sqnorm_and_adam_update."""
    g = DK._gen(seed * 100003 + i)
    sign = lambda: torch.where(torch.rand(length, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    logu = lambda lo, hi: torch.exp(torch.empty(length, device=DEV).uniform_(math.log(lo), math.log(hi), generator=g))
    p = torch.randn(length, generator=g, device=DEV) * 0.05
    gr = sign() * logu(1e-8, 1e-3)
    m = sign() * logu(1e-9, 1e-4)
    v = logu(1e-18, 1e-8)
    return p, gr, m, v


def test_flat_casts_and_split_past_2_31_elements(ops):
    n = N_FLAT
    need(n * 8 / GIB + 0.5, f"casts n={n} (f32 source, bf16 hi and lo, then bf16 -> f32: {n * 8 / GIB:.1f} GiB)")
    src = guarded((n,), F32, fill=None)
    for i, a, b in flat_slabs(n):
        src.out[a:b] = torch.randn(b - a, generator=DK._gen(7 * 100003 + i), device=DEV) * 4.0
    hi, lo = guarded((n,), BF16), guarded((n,), BF16)
    ops.cast_f32_to_bf16(src.out, hi.out)
    for i, a, b in checked_slabs(n):
        x = torch.randn(b - a, generator=DK._gen(7 * 100003 + i), device=DEV) * 4.0
        exact(f"cast_f32_to_bf16 n=2^31+37 [{a}, {b})", hi.out[a:b], x.to(BF16))
    assert_untouched("cast_f32_to_bf16", hi)
    hi.out.fill_(math.nan)
    ops.split_f32(src.out, hi.out, lo.out)
    for i, a, b in checked_slabs(n):
        x = torch.randn(b - a, generator=DK._gen(7 * 100003 + i), device=DEV) * 4.0
        h = x.to(BF16)
        exact(f"split_f32 hi n=2^31+37 [{a}, {b})", hi.out[a:b], h)
        exact(f"split_f32 lo n=2^31+37 [{a}, {b})", lo.out[a:b], (x - h.float()).to(BF16))
    assert_untouched("split_f32 hi", hi)
    assert_untouched("split_f32 lo", lo)
    assert_untouched("cast source", src)
    del src, lo
    torch.cuda.empty_cache()
    wide = guarded((n,), F32)
    ops.cast_bf16_to_f32(hi.out, wide.out)
    for i, a, b in checked_slabs(n):
        x = torch.randn(b - a, generator=DK._gen(7 * 100003 + i), device=DEV) * 4.0
        exact(f"cast_bf16_to_f32 n=2^31+37 [{a}, {b})", wide.out[a:b], x.to(BF16).float())
    assert_untouched("cast_bf16_to_f32", wide)


def test_sqnorm_and_adam_past_2_31_elements(ops):
    """sqnorm of g, then adam_step with the clip active, weight decay, the bf16 shadow and zero_grad, n = 2^31 + 37."""
    n = N_FLAT
    gib = n * 18 / GIB
    need(gib + 2.0, f"sqnorm + adam n={n} (p, m, v, g f32 and the bf16 shadow: {gib:.1f} GiB + 2 GiB of checks)")
    seed = 11
    bufs = {k: guarded((n,), F32, fill=None) for k in ("p", "g", "m", "v")}
    for i, a, b in flat_slabs(n):
        for k, t in zip(("p", "g", "m", "v"), adam_inputs(seed, i, b - a)):
            bufs[k].out[a:b] = t
    gn_base = 1e-3
    gn = torch.full((1,), gn_base, device=DEV)
    ops.sqnorm(bufs["g"].out, gn)
    sq = torch.zeros((), dtype=F64, device=DEV)
    for _, a, b in flat_slabs(n):
        sq += (bufs["g"].out[a:b].to(F64) ** 2).sum()
    sq = gn_base + sq
    blocks = min(-(-(n // 4) // 256), 8 * DK._sm())
    depth = 4 * -(-(n // 4) // (blocks * 256)) + 5 + 8 + blocks + 8
    DK.check("sqnorm n=2^31+37", gn, sq.reshape(1), sq.reshape(1), a=0.0, b=depth * U)
    p16 = guarded((n,), BF16)
    lr, b1, b2, eps, wd, clip = 1e-3, 0.9, 0.999, 1e-6, 0.01, 1.0
    ops.adam_step(bufs["p"].out, bufs["m"].out, bufs["v"].out, bufs["g"].out, p16.out, lr, b1, b2, eps, wd, gn, clip,
                  1.0, False, 0, zero_grad=True)
    for i, a, b in checked_slabs(n):
        p, gr, m, v = adam_inputs(seed, i, b - a)
        clipped = DK.check_adam_update(f"n=2^31+37 [{a}, {b})", (p, m, v, gr, gn),
                                       tuple(t.out[a:b] for t in (bufs["p"], bufs["m"], bufs["v"], p16)),
                                       lr, b1, b2, eps, wd, clip, 1.0, False, 0)
        assert clipped
    for _, a, b in flat_slabs(n):
        assert bool((bufs["g"].out[a:b] == 0).all()), f"zero_grad left [{a}, {b}) non-zero"
    for k, t in list(bufs.items()) + [("p_bf16", p16)]:
        assert_untouched(f"adam {k}", t)


# ------------------------------------------------------------------------------------------------------- A: input image
def test_image_crop_at_a_byte_offset_above_2_32(ops):
    from oracle import data as odata
    H, W, C, size = 300, 211, 3, 256
    off = 2 ** 32 + 4097                           # odd
    total = off + H * W * C + 1001
    need(total / GIB + 0.5, f"crop_resize in a {total / 1e9:.1f} GB buffer")
    rng = np.random.default_rng(3)
    imgs = [rng.integers(0, 256, (H, W, C), dtype=np.uint8) for _ in range(2)]
    packed = torch.randint(0, 256, (total,), dtype=torch.uint8, device=DEV, generator=DK._gen(5))
    offsets = [off - 2 ** 32, off]                 # the second image's offset truncated to 32 bits is the first's
    for im, o in zip(imgs, offsets):
        packed[o:o + im.size] = torch.from_numpy(im.reshape(-1)).to(DEV)
    out = guarded((2, size, size, C), F32)
    ops.image_crop_resize_normalize(packed, torch.tensor(offsets, dtype=torch.int64, device=DEV),
                                    torch.full((2,), H, dtype=I32, device=DEV), torch.full((2,), W, dtype=I32, device=DEV),
                                    torch.from_numpy(np.stack([odata.reference_crop_box(H, W)] * 2)).to(DEV), out.out,
                                    C, size)
    for k, im in enumerate(imgs):
        want = torch.from_numpy(odata.decode_img(im, size)).to(DEV)
        exact(f"image_crop_resize_normalize image at byte offset {offsets[k]}", out.out[k], want)
    assert_untouched("image_crop_resize_normalize", out)


# ------------------------------------------------------------------------------------------------------- B: dropout
def _elem_drop(site, rate=0.1):
    from dalle_mtf_b200 import lib as L
    return L.make_dropout(rate, 9, 4, site, ELEM_ROW0)


def test_dropout_masks_with_the_counter_high_word_set(ops):
    from dalle_mtf_b200 import lib as L
    from oracle import philox as X
    e0 = ELEM_ROW0 * ELEM_COLS
    assert (e0 >> 2) < 2 ** 32 <= (e0 + ELEM_ROWS * ELEM_COLS - 1) >> 2
    site = L.dropout_site_mlp_out(0)
    keep = torch.empty(ELEM_ROWS, ELEM_COLS, dtype=torch.uint8, device=DEV)
    ops.dropout_mask(_elem_drop(site), L.DROPOUT_ELEMENTWISE, (ELEM_ROWS, ELEM_COLS), keep)
    want = X.keep_elementwise(0.1, 9, 4, site, ELEM_ROWS, ELEM_COLS, ELEM_ROW0)
    exact(f"dropout_mask elementwise row0=2^25-3 cols={ELEM_COLS}", keep, torch.from_numpy(want.astype(np.uint8)).to(DEV))
    S2 = (ATTN_S + 1) // 2
    assert ((ATTN_ROW0 * ATTN_H + 21) * S2) * S2 < 2 ** 32 <= ((ATTN_ROW0 * ATTN_H + 22) * S2) * S2 - 1
    drop = L.make_dropout(0.1, 5, 11, L.dropout_site_attn(0), ATTN_ROW0)
    keep = torch.empty(ATTN_B, ATTN_H, ATTN_S, ATTN_S, dtype=torch.uint8, device=DEV)
    ops.dropout_mask(drop, L.DROPOUT_ATTENTION, (ATTN_B, ATTN_H, ATTN_S), keep)
    for b in range(ATTN_B):                        # one sequence at a time: the oracle's uint64 temporaries are large
        want = X.keep_attention(0.1, 5, 11, L.dropout_site_attn(0), 1, ATTN_H, ATTN_S, ATTN_ROW0 + b)[0]
        exact(f"dropout_mask attention sequence {ATTN_ROW0 + b} H={ATTN_H} S={ATTN_S}", keep[b],
              torch.from_numpy(want.astype(np.uint8)).to(DEV))


def test_gemm_store_residual_dropout_with_the_counter_high_word_set(ops):
    from dalle_mtf_b200 import lib as L
    M, N, K = ELEM_ROWS, ELEM_COLS, 512
    # the engine's attention-output product: bias + residual, residual dropout in the STORE epilogue
    desc = ("gemm", M, N, K, False, True, L.EPI_STORE, "torch.bfloat16", True, False, True, False, 1, 0, False, True)
    DK.run_gemm_case(ops, desc, M, M, seed=3, dropout=_elem_drop(L.dropout_site_attn_out(0)), tag="row0=2^25-3 ")


def test_layernorm_backward_dropout_with_the_counter_high_word_set(ops):
    from dalle_mtf_b200 import lib as L
    DK.run_layernorm(ops, f"LN dropout rows={ELEM_ROWS} d={ELEM_COLS} row0=2^25-3", ELEM_ROWS, ELEM_COLS,
                     dropout=_elem_drop(L.dropout_site_mlp_out(0)), seed=5)


def test_embedding_dropout_with_the_counter_high_word_set(ops):
    from dalle_mtf_b200 import lib as L
    V = 50771
    g = DK._gen(17)
    ids = torch.randint(0, V, (1, ELEM_ROWS), generator=g, device=DEV, dtype=I32)
    ids[0, 2:5] = 7                                # a run of equal ids straddling the high-word row
    DK.run_embedding(ops, f"embedding dropout tokens={ELEM_ROWS} d={ELEM_COLS} row0=2^25-3", ids, V, ELEM_COLS, 1.0, g,
                     wte_drop=_elem_drop(L.SITE_WTE, 0.25), wpe_drop=L.make_dropout(0.25, 9, 4, L.SITE_WPE, 0))


def test_attention_dropout_with_the_counter_high_word_set(ops):
    from dalle_mtf_b200 import lib as L
    B, S, H, dh = ATTN_B, ATTN_S, ATTN_H, ATTN_DH
    need(6.0, f"attention dropout B={B} H={H} S={S} (float64 references of one sequence)")
    qkv, dout = DK._qkv(B, S, H, dh, DK._gen(B * H + 1))
    drop = L.make_dropout(0.1, 5, 11, L.dropout_site_attn(0), ATTN_ROW0)
    DK.run_attention(ops, f"attention dropout B={B} S={S} H={H} dh={dh} row0={ATTN_ROW0}", B, S, H, dh, 1.0, qkv, dout,
                     dropout=drop)


def test_caption_dropout_with_the_counter_high_word_set(ops):
    from dalle_mtf_b200 import lib as L
    from oracle import guidance as CG
    assert (CAP_ROW0 >> 2) < 2 ** 32 <= (CAP_ROW0 + CAP_B - 1) >> 2
    g = torch.Generator().manual_seed(1)
    Tt, Ti, tv, pad = 256, 1024, 50258, 50257
    text = torch.randint(0, pad, (CAP_B, Tt), generator=g, dtype=I32)
    img = torch.randint(0, 512, (CAP_B, Ti), generator=g, dtype=I32)
    out = torch.full((CAP_B, Tt + Ti), -1, dtype=I32, device=DEV)
    rate, seed, step = 0.5, 2 ** 40 + 3, 17
    ops.assemble_tokens(text.to(DEV), img.to(DEV), out, tv, caption_drop=L.make_dropout(rate, seed, step,
                                                                                          L.SITE_CAPTION, CAP_ROW0),
                        pad_id=pad)
    dropped = torch.from_numpy(CG.caption_dropped(rate, seed, step, CAP_B, CAP_ROW0))
    want = torch.cat([text, img + tv], 1)
    want[dropped, :Tt] = pad
    assert 0 < int(dropped.sum()) < CAP_B
    exact(f"assemble_tokens_ex caption dropout row0=2^34-5 B={CAP_B}", out, want.to(DEV))


# ------------------------------------------------------------------------------------------------------- C: samplers
@pytest.mark.parametrize("n", [32769, 50771, 51200])
@pytest.mark.parametrize("rows", [1, 33])
def test_filtered_sampler_at_the_widest_rows(ops, rows, n):
    SF.check_filtered_rows(ops, rows, n)
    print(f"[{TAG}] sample_rows_filtered rows={rows} n={n}: kept counts and draws equal the oracle's "
          "(worst err/bound 0)")


@pytest.mark.parametrize("n", [32769, 50771, 51200])
@pytest.mark.parametrize("rows", [1, 33])
def test_guided_sampler_at_the_widest_rows(ops, rows, n):
    GU.check_guided_rows(ops, rows, n)
    print(f"[{TAG}] sample_rows_guided rows={rows} n={n}: kept counts and draws equal the oracle's "
          "(worst err/bound 0)")


def test_one_id_past_the_filtered_limit_is_rejected_before_any_launch(ops):
    from dalle_mtf_b200 import lib as L
    lib, s = L.load(), torch.cuda.current_stream().cuda_stream
    lo, n = 3, 51201
    logits = torch.randn(2, lo + n + 1, device=DEV)
    idx = torch.full((2,), -1, dtype=I32, device=DEV)
    kept = torch.full((2,), -1, dtype=I32, device=DEV)
    torch.cuda.synchronize()
    before = lib.db200_launch_count()
    rc = lib.db200_sample_rows_filtered(s, logits.data_ptr(), None, idx.data_ptr(), kept.data_ptr(), 2,
                                        logits.stride(0), lo, lo + n, 1.0, 8, 0.9)
    assert rc == -4, rc                                                   # DB200_E_UNSUPPORTED
    tokens = torch.full((2, 2), -1, dtype=I32, device=DEV)
    rc = lib.db200_sample_rows_guided(s, logits.data_ptr(), logits.stride(0), None, tokens.data_ptr(), 2,
                                      kept.data_ptr(), 1, lo, lo + n, 1.0, 3.0, 8, 0.9, None)
    assert rc == -4, rc
    torch.cuda.synchronize()
    assert lib.db200_launch_count() == before
    assert (idx == -1).all() and (kept == -1).all() and (tokens == -1).all()
    print(f"[{TAG}] n={n}: DB200_E_UNSUPPORTED, no launch (worst err/bound 0)")


@pytest.mark.parametrize("rows", [1, 33])
def test_unfiltered_sampler_at_58496_ids(ops, rows):
    """sample_rows has no width limit: greedy is the first maximum (ties planted at two ids), with noise the first
    Gumbel-max."""
    n, lo = 58496, 9
    hi, ld = lo + n, lo + n + 7
    g = DK._gen(rows + n)
    logits = torch.randn(rows, ld, generator=g, device=DEV) * 3
    logits[:, lo + 1000] = logits[:, lo + n - 1] = 30.0                 # ties of the maximum: the first one wins
    logits[::2, lo + n - 1] = 31.0                                      # the maximum at the last id
    logits[:, :lo] = logits[:, hi:] = 100.0                             # outside [lo, hi): never selected
    idx = torch.empty(rows, dtype=I32, device=DEV)
    ops.sample_rows(logits, None, idx, lo, hi, 1.0)
    want = (logits[:, lo:hi].argmax(-1) + lo).to(I32)
    exact(f"sample_rows greedy rows={rows} n={n}", idx, want)
    u = torch.empty(rows, n, device=DEV).uniform_(1e-9, 1.0, generator=g)
    ops.sample_rows(logits, u, idx, lo, hi, 1.0)
    mask = np.ones((rows, n), dtype=bool)
    SF.check_selection(idx.cpu().long(), lo, mask, SF.perturbed(logits[:, lo:hi], u, 1.0), np.ones(rows, dtype=bool))
    print(f"[{TAG}] sample_rows with noise rows={rows} n={n}: a first Gumbel-max (worst err/bound 0)")
