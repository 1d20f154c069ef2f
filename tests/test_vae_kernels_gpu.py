"""Discrete-VAE kernels against float64 references of the same operation on the same operands.

Every case feeds a kernel and a float64 torch computation (on the GPU) the SAME operands: where a kernel consumes
rounded values (bf16 activations, the tensor-core convolutions' bf16 weights, the first layer's hi + lo split image,
the codebook's hi + lo parts) the reference is given exactly those values, so the only difference left is the kernel's
own arithmetic.  Each output element must satisfy

    |got - ref| <= a * |ref| + b * absref

where absref is the same operation in float64 on |operands| (conv(|x|, |w|), |y| @ |C|^T, ...), which bounds every
partial sum the kernel can form.

  a  output rounding.  fp32 outputs: a few u, u = 2^-24.  bf16 outputs: half an ulp of bf16 at |ref| (<= 2^-8 |ref|)
     instead of a * |ref|, so a kernel that loses low-order bits is not hidden by a value that rounds favourably.
  b  accumulation over the case's contraction length L: L roundings of a partial sum, each <= u_acc * absref (the
     classical worst-case bound gamma_L).  u_acc = 2^-24 for fp32 FMA chains and 2^-23 for wgmma accumulation (the
     tensor core may truncate instead of rounding).  The fp32 convolutions / rowmatmul on wgmma add six split
     products per term (conv_f32_tc.cu), so they take 6 L steps.  Split-K, atomics and epilogue adds (bias, residual,
     accumulate-into) add a handful of steps, covered by + 8 u.
  split terms (codebook on wgmma, vae_engine.py _mm_split): x = hi + lo + e with |lo| <= 2^-8 |x| and
     |e| <= 2^-16 |x|.  One exact bf16 operand times a split one drops hi*e_c: SPLIT1 = 1.01 * 2^-16.  Two split
     operands (three products, lo*lo dropped) drop lo*lo, hi*e_c, e_x*hi and smaller: SPLIT2 = 3.1 * 2^-16.
  Gumbel softmax: z = (l - log(-log u)) / tau carries an absolute error <= 2^-21 (1 + |l| + |g|) / tau (two logf and
     three roundings), and z_k - max z one more rounding; exp(.) turns absolute errors of the exponent into relative
     errors of y, the normalising sum adds (K/32 + 8) u, expf and the division 2^-20.  Outputs that underflow to
     fp32 subnormals get an absolute floor of 2^-148.

Outputs a kernel writes are filled with NaN first, so an element it never writes fails; outputs it accumulates into
(dw, dbias, rowmatmul_tn, rowmatmul accumulate=1, the mse loss, the codebook gradient) start from a non-zero base that
the reference adds too, so a kernel that overwrites instead of adding fails.  One `[vae-kernels]` line per case gives
the worst err/bound ratio (must be < 1).  bf16 cases with a short contraction report ratios just below 1: among
millions of outputs some lie within b * absref of a rounding midpoint, where the half-ulp term is all the slack there is.

The wgmma convolutions run at the geometry of the two VAE configurations, at a batch chosen so that every launch has at
least twice as many work tiles as the device has SMs (the persistent CTAs then walk several tiles each), and at edge
geometries: ragged spatial sizes, several images packed into one tile, 64-wide and ragged channel tiles, 1x1 kernels
(one k-block per tile at 64 input channels), and a wgrad with fewer pixel tiles than the split count the host rule
asks for.  Each check also runs a mutated reference that must fail (run_conv).
"""
import functools
import json
import math
import os

import pytest
import torch

import float64_bounds
from float64_bounds import DEV, NAN, U, UTC, nan_like

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
check = functools.partial(float64_bounds.check, tag="vae-kernels")

SPLIT1 = 1.01 * 2.0 ** -16
SPLIT2 = 3.1 * 2.0 ** -16


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def _sm():
    return float64_bounds.sm_count()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, g, scale=1.0, dtype=F32):
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def first_argmax(x):
    """Lowest index of the row maximum (tf.math.argmax / np.argmax), independent of torch's tie behaviour."""
    m = x.max(-1, keepdim=True).values
    k = torch.arange(x.shape[-1], device=x.device).expand_as(x)
    return torch.where(x == m, k, x.shape[-1]).min(-1).values


# ------------------------------------------------------------------------------------------------------- tile rules
def _pow2_floor(x):
    p = 1
    while p * 2 <= x:
        p *= 2
    return p


def choose_tile(OW, OH):
    """conv_tc.cu choose_tile: a 128-pixel tile of TN images x TH rows x TW columns."""
    TW = _pow2_floor(min(OW, 16))
    TH = _pow2_floor(min(OH, 128 // TW))
    return TW, TH, 128 // (TW * TH)


def gather_tiles(N, OH, OW, Nn):
    """Work tiles of one conv_tc_kernel launch (run_gather): pixel tiles x channel tiles."""
    TW, TH, TN = choose_tile(OW, OH)
    bn = 128 if Nn >= 128 else 64
    return -(-N // TN) * -(-OH // TH) * -(-OW // TW) * -(-Nn // bn)


def out_res(H, stride, transposed):
    return 2 * H if transposed else -(-H // stride)


def tc_tiles(N, H, Cin, Cout, stride, transposed):
    """(forward, dgrad) tiles per wgmma launch; strided scatters run one launch per output parity."""
    Ho = out_res(H, stride, transposed)
    fwd = gather_tiles(N, H, H, Cout) if transposed else gather_tiles(N, Ho, Ho, Cout)
    dg = gather_tiles(N, H // 2, H // 2, Cin) if (stride == 2 and not transposed) else gather_tiles(N, H, H, Cin)
    return fwd, dg


def wgrad_split(N, H, Cin, Cout, k, stride, transposed, sm):
    """conv2d_wgrad_tc's host rule: (pixel tiles, splits the SM count asks for, splits used, pixel tiles per split)."""
    OH = H if transposed else out_res(H, stride, transposed)
    TW, TH, TN = choose_tile(OH, OH)
    ptiles = -(-N // TN) * -(-OH // TH) * -(-OH // TW)
    items = -(-Cin // 128) * -(-Cout // (128 if Cout >= 128 else 64)) * k * k
    wanted = -(-2 * sm // items)
    splits = max(min(wanted, ptiles), 1)
    per = -(-ptiles // splits)
    return ptiles, wanted, -(-ptiles // per), per


# ------------------------------------------------------------------------------------------------------- convolutions
def _conv64(x, w, stride, transposed):
    from oracle import vae as OV
    return OV.conv2d_transpose_same(x, w, None) if transposed else OV.conv2d_same(x, w, None, stride)


def conv_refs(x, w, dy, stride, transposed):
    """float64 (y, dx, dw) of the convolution on (x, w, dy) and on (|x|, |w|, |dy|)."""
    out = []
    for xx, ww, gg in ((x, w, dy), (x.abs(), w.abs(), dy.abs())):
        xx = xx.to(F64).requires_grad_(True)
        ww = ww.to(F64).requires_grad_(True)
        y = _conv64(xx, ww, stride, transposed)
        dx, dw = torch.autograd.grad(y, (xx, ww), gg.to(F64))
        out.append((y.detach(), dx, dw))
    return out


FWD_VARIANTS = ("plain", "relu", "res")
DGRAD_VARIANTS = ("plain", "mask", "dres", "dres in place", "mask dres in place")
WGRAD_REL = 2.0 ** -12


def must_fail(name, got, wrong_ref, absref, **bound):
    """A reference with one deliberate mistake (a mutation) must be told apart from the kernel's output."""
    r = float64_bounds.worst_ratio(name, got, wrong_ref, absref, **bound)
    assert r >= 1.0, f"{name}: the mutated reference passes too (worst err/bound {r:.4f})"


def _mask_operand(shape, g, dtype):
    """A ReLU mask as the engine passes it: a post-ReLU activation or a block input, with exact zeros and
    negatives (only > 0 keeps the gradient)."""
    m = _randn(*shape, g=g, dtype=dtype)
    m.view(-1)[::5] = 0
    return m


def run_conv(ops, tag, N, H, Cin, Cout, k, stride, transposed, *, dgrad=True, wgrad=True, res_block=False,
             act_f32=False, seed=0, fwd_variants=None, dgrad_variants=None, line_tag="vae-kernels"):
    """Forward, dgrad and wgrad (+ bias gradient) of one convolution through the kernels VaeEngine picks for it,
    with the arguments the engine passes: a residual block's conv_in runs with the fused ReLU, its conv_out with the
    residual add; their dgrads with the ReLU mask (conv_out) and the residual gradient (conv_in), which the engine
    reads from and writes to the same buffer (VaeEngine._res_bwd).  PaperVaeEngine also passes the mask and the
    in-place residual gradient in one launch (_block_bwd).  fwd_variants / dgrad_variants (names from FWD_VARIANTS /
    DGRAD_VARIANTS) replace those sets by the ones an engine was seen to launch; wgrad=False skips the weight
    gradient (a forward-only launch).

    Every check also runs a mutated reference that must fail: the mask or the residual gradient dropped, a 1x1
    output compared one pixel over, the weight gradient without its base."""
    g = _gen(seed)
    act = F32 if act_f32 else BF16
    chk = functools.partial(float64_bounds.check, tag=line_tag)
    if fwd_variants is None:
        fwd_variants = ("relu", "res") if res_block else ("plain",)
    if dgrad_variants is None:
        dgrad_variants = ("mask", "dres", "dres in place", "mask dres in place") if res_block else ("plain",)
    assert set(fwd_variants) <= set(FWD_VARIANTS) and set(dgrad_variants) <= set(DGRAD_VARIANTS)
    Ho = out_res(H, stride, transposed)
    wshape = (k, k, Cout, Cin) if transposed else (k, k, Cin, Cout)
    x = _randn(N, H, H, Cin, g=g, dtype=act)
    # fp32 weights: full fp32 values for the fp32 kernels, bf16-exact values otherwise (the wgmma kernels read the
    # engine's bf16 shadow, the direct kernels the fp32 master of the same bf16 weights)
    w = _randn(*wshape, g=g, scale=(k * k * Cin) ** -0.5)
    if not act_f32:
        w = w.to(BF16).float()
    w16 = w.to(BF16)
    bias = _randn(Cout, g=g, scale=0.1)
    dy = _randn(N, Ho, Ho, Cout, g=g, dtype=act)
    (y64, dx64, dw64), (ya, dxa, dwa) = conv_refs(x, w, dy, stride, transposed)
    c = ops.conv_desc(N, H, H, Cin, Cout, k, k, stride, transposed=transposed, act_f32=act_f32)
    c_relu = ops.conv_desc(N, H, H, Cin, Cout, k, k, stride, transposed=transposed, act_f32=act_f32, relu=True)
    fwd_tc = ops.conv_tc_supported(c)          # False for fp32 descriptors
    dg_tc = ops.conv_dgrad_tc_supported(c)
    wg_tc = ops.conv_wgrad_tc_supported(c)
    u_acc = 6 * UTC if act_f32 else UTC
    taps_per_out = 4 if transposed else k * k
    L_f, L_d, L_w = taps_per_out * Cin, k * k * Cout, N * (H * H if transposed else Ho * Ho)
    kind = "f32" if act_f32 else "bf16"
    ratios = []

    # ---- forward
    for label in fwd_variants:
        relu = label == "relu"
        res = _randn(N, Ho, Ho, Cout, g=g, dtype=act) if label == "res" else None
        y = nan_like((N, Ho, Ho, Cout), act)
        cc = c_relu if relu else c
        if fwd_tc:
            ops.conv2d_fwd_tc(cc, x, w16, bias, res, y)
        else:
            ops.conv2d_fwd(cc, x, w, bias, res, y)
        ref = y64 + bias.to(F64)
        absref = ya + bias.abs().to(F64)
        if relu:
            ref = ref.clamp_min(0)
        if res is not None:
            ref = ref + res.to(F64)
            absref = absref + res.abs().to(F64)
        name = f"{tag} fwd {label} [{'wgmma' if fwd_tc else 'direct'} {kind}]"
        bound = dict(b=L_f * u_acc + 8 * U, bf16_out=not act_f32)
        ratios.append(chk(name, y, ref, absref, **bound))
        if k == 1:
            must_fail(name + " one pixel over", y, ref.roll(1, 2), absref.roll(1, 2), **bound)

    # ---- dgrad
    for label in dgrad_variants if dgrad else ():
        mask = _mask_operand((N, H, H, Cin), g, act) if "mask" in label else None
        dres = _randn(N, H, H, Cin, g=g, dtype=act) if "dres" in label else None
        in_place = "in place" in label
        dx = dres.clone() if in_place else nan_like((N, H, H, Cin), act)
        dres_arg = dx if in_place else dres
        if dg_tc:
            ops.conv2d_dgrad_tc(c, dy, w16, mask, dres_arg, dx)
        else:
            ops.conv2d_dgrad(c, dy, w, mask, dres_arg, dx)
        ref, absref = dx64, dxa
        keep = (mask > 0).to(F64) if mask is not None else 1.0
        add, add_abs = (dres.to(F64), dres.abs().to(F64)) if dres is not None else (0.0, 0.0)
        name = f"{tag} dgrad {label} [{'wgmma' if dg_tc else 'direct'} {kind}]"
        bound = dict(b=L_d * u_acc + 8 * U, bf16_out=not act_f32)
        ratios.append(chk(name, dx, ref * keep + add, absref * keep + add_abs, **bound))
        if mask is not None:
            must_fail(name + " mask dropped", dx, ref + add, absref + add_abs, **bound)
        if dres is not None:
            must_fail(name + " dres dropped", dx, ref * keep, absref * keep, **bound)

    # ---- wgrad + bias gradient, accumulated onto non-zero bases.  The componentwise bound grows as L_w while the
    # gradient grows as sqrt(L_w): past L_w ~ 2^16 it exceeds the gradient itself.  So the base is made larger than the
    # bound (a kernel that drops it still fails), and the gradient (dw - base) is also held to a relative Frobenius
    # error of WGRAD_REL, which a lost pixel tile or split exceeds.
    if not wgrad:        # a forward-only launch (the tokenizer)
        return ratios
    b_w = (L_w + 64) * u_acc + 8 * U
    assert b_w < 0.5, (tag, L_w)
    base_w = _randn(*wshape, g=g, scale=max(math.sqrt(L_w), 4 * b_w * float(dwa.max()) / (1 - b_w)))
    base_b = _randn(Cout, g=g, scale=math.sqrt(L_w))
    dw, db = base_w.clone(), base_b.clone()
    if wg_tc:
        ops.conv2d_wgrad_tc(c, x, dy, dw)
        ops.colsum(dy.view(-1, Cout), db)
    else:
        ops.conv2d_wgrad(c, x, dy, dw, db)
    wlabel = "wgmma" if wg_tc else "direct"
    name = f"{tag} wgrad [{wlabel} {kind}]"
    ratios.append(chk(name, dw, base_w.to(F64) + dw64, base_w.abs().to(F64) + dwa, b=b_w))
    must_fail(name + " without its base", dw, dw64, base_w.abs().to(F64) + dwa, b=b_w)
    rel = ((dw.to(F64) - base_w.to(F64) - dw64).norm() / dw64.norm().clamp_min(1e-300)).item()
    assert rel < WGRAD_REL, f"{name}: relative Frobenius error {rel:.3g} of dw - base"
    dy64 = dy.to(F64).reshape(-1, Cout)
    ratios.append(chk(f"{tag} dbias [{'colsum' if wg_tc else 'direct'} {kind}]", db,
                      base_b.to(F64) + dy64.sum(0), base_b.abs().to(F64) + dy64.abs().sum(0),
                      b=(L_w + 64) * 2 * U + 8 * U))
    return ratios


def _config(name):
    with open(os.path.join(ROOT, "configs", name + ".json")) as f:
        return json.load(f)


def _engine(name):
    from dalle_mtf_b200.vae_engine import VaeEngine
    cfg = _config(name)
    return VaeEngine(cfg["num_tokens"], cfg["dataset"]["image_size"], cfg["convblocks"], use_bf16=True)


def engine_convs(eng):
    """Every distinct convolution of the engine's training step, read from its layer lists:
    (kind, Cin, Cout, res, k, stride, transposed, dgrad_needed)."""
    seen = {}
    for li, (kind, _, cin, ch, res) in enumerate(eng.enc):
        key = ("down", cin, ch, res, 4, 2, False, li > 0) if kind == "down" else ("res", ch, ch, res, 3, 1, False, True)
        seen.setdefault(key, None)
    for kind, _, cin, ch, res in eng.dec:
        key = ("up", cin, ch, res, 4, 2, True, True) if kind == "up" else ("res", ch, ch, res, 3, 1, False, True)
        seen.setdefault(key, None)
    seen.setdefault(("out", eng.dec_out_cin, eng.C, eng.H, 1, 1, False, True), None)
    return list(seen)


def production_batch(ops, kind, cin, cout, res, k, stride, transposed, dgrad, sm):
    """Smallest batch at which every wgmma launch of this layer has >= 2 x SM work tiles (2 for the direct kernels)."""
    c = ops.conv_desc(1, res, res, cin, cout, k, k, stride, transposed=transposed, act_f32=False)
    used = (ops.conv_tc_supported(c), dgrad and ops.conv_dgrad_tc_supported(c))
    if not any(used) and not ops.conv_wgrad_tc_supported(c):
        return 2
    for n in range(1, 1025):
        tiles = tc_tiles(n, res, cin, cout, stride, transposed)
        if all(t >= 2 * sm for t, u in zip(tiles, used) if u):
            return n
    raise AssertionError("no batch reaches 2 x SM tiles")


@pytest.mark.parametrize("config", ["vae_example_b200", "vae_coco_b200"])
def test_convolutions_at_the_production_geometry(ops, config):
    production_convolutions(ops, config)


def production_convolutions(ops, config, several_splits=True):
    """run_conv (bf16, and fp32 at a quarter of the batch) on every convolution of the configuration's training step,
    at the batch production_batch() picks for the current SM count.  several_splits: every pixel-split wgrad must run
    several splits of several pixel tiles (true of these geometries on a 132-SM H100; with fewer SMs, vae_coco's
    512-channel layers ask for a single split).  Returns (layer, batch) per layer."""
    eng = _engine(config)
    sm = _sm()
    layers = engine_convs(eng)
    assert any(kind == "up" for kind, *_ in layers) and any(kind == "res" for kind, *_ in layers)
    worst = 0.0
    batches = []
    for i, (kind, cin, cout, res, k, stride, transposed, dgrad) in enumerate(layers):
        n = production_batch(ops, kind, cin, cout, res, k, stride, transposed, dgrad, sm)
        batches.append((layers[i], n))
        c = ops.conv_desc(n, res, res, cin, cout, k, k, stride, transposed=transposed, act_f32=False)
        fwd_t, dg_t = tc_tiles(n, res, cin, cout, stride, transposed)
        if ops.conv_tc_supported(c):
            assert fwd_t >= 2 * sm, (kind, cin, cout, res, n, fwd_t)
        if dgrad and ops.conv_dgrad_tc_supported(c):
            assert dg_t >= 2 * sm, (kind, cin, cout, res, n, dg_t)
        if several_splits and ops.conv_wgrad_tc_supported(c):   # several splits, each over several pixel tiles
            _, _, splits, per = wgrad_split(n, res, cin, cout, k, stride, transposed, sm)
            assert splits >= 2 and per >= 2, (kind, cin, cout, res, n, splits, per)
        tag = f"{config} {kind} {cin}->{cout} @{res} N={n}"
        worst = max([worst] + run_conv(ops, tag, n, res, cin, cout, k, stride, transposed, dgrad=dgrad,
                                       res_block=kind == "res", seed=i))
        # the fp32 kernels (fp32-activation engines) on the same descriptor at a smaller batch
        nf = max(1, n // 4)
        worst = max([worst] + run_conv(ops, f"{config} {kind} {cin}->{cout} @{res} N={nf}", nf, res, cin, cout, k,
                                       stride, transposed, dgrad=dgrad, res_block=kind == "res", act_f32=True,
                                       seed=100 + i))
    print(f"{float64_bounds.prefix()}[vae-kernels] {config} convolutions: worst err/bound {worst:.4f}")
    return batches


EDGE_GEOMETRIES = [
    (3, 12, 64, 64, 3, 1, False),      # 12 px: tiles run past the image edge
    (2, 20, 64, 192, 3, 1, False),     # 20 px; Cout 192: the second 128-wide channel tile is half empty
    (2, 24, 128, 64, 4, 2, False),     # stride 2, 24 -> 12; 64-wide channel tile
    (3, 12, 64, 192, 4, 2, True),      # conv-transpose 12 -> 24, ragged channel tile
    (5, 8, 64, 128, 3, 1, False),      # 8 px: two images per tile, N odd
    (13, 4, 128, 64, 3, 1, False),     # 4 px: eight images per tile, N = 13
    (13, 8, 64, 64, 4, 2, False),      # stride 2 onto 4 px: eight images per tile; dgrad gathers 4 px parities
    (7, 4, 64, 64, 4, 2, True),        # conv-transpose from 4 px: eight images per tile, N = 7
    (1, 8, 64, 64, 3, 1, False),       # wgrad: one pixel tile, fewer than the splits the SM count asks for
    (3, 8, 128, 128, 4, 2, False),     # wgrad over 4 px outputs, 3 images per 8-image tile
    (6, 16, 64, 256, 1, 1, False),     # 1x1, Cin 64: one k-block per tile, the stage ring wraps every four tiles
    (3, 12, 192, 192, 1, 1, False),    # 1x1, 12 px; 192 channels: ragged last channel tile on both sides
    (3, 32, 128, 64, 1, 1, False),     # 1x1 at 32 px (the token grid): 64-wide output channel tile
    (13, 4, 64, 128, 1, 1, False),     # 1x1 at 4 px: eight images per tile, N = 13
]


@pytest.mark.parametrize("N,H,Cin,Cout,k,stride,transposed", EDGE_GEOMETRIES)
def test_tensor_core_convolutions_at_edge_geometries(ops, N, H, Cin, Cout, k, stride, transposed):
    c = ops.conv_desc(N, H, H, Cin, Cout, k, k, stride, transposed=transposed, act_f32=False)
    assert ops.conv_tc_supported(c) and ops.conv_dgrad_tc_supported(c) and ops.conv_wgrad_tc_supported(c)
    ptiles, wanted, splits, per = wgrad_split(N, H, Cin, Cout, k, stride, transposed, _sm())
    if (N, H) == (1, 8):
        assert ptiles < wanted and splits == ptiles == 1
    run_conv(ops, f"edge N={N} {H}px {Cin}->{Cout} k{k} s{stride}{' T' if transposed else ''}", N, H, Cin, Cout, k,
             stride, transposed, res_block=not transposed and stride == 1, seed=N * 1000 + H)


# ------------------------------------------------------------------------------------------------------- first layer
@pytest.mark.parametrize("N,H,W,Cout", [(32, 256, 256, 64), (32, 256, 256, 128), (3, 34, 34, 64), (2, 18, 50, 128)])
@pytest.mark.parametrize("kernel", ["wgmma", "fma"])
def test_first_layer_convolution(ops, N, H, W, Cout, kernel):
    """conv2d_first_fwd (wgmma) sees the image as bf16 hi + lo and the weights as bf16; the fma kernel sees both in
    fp32.  The reference gets the same operands.  Dropping the lo half of the image moves elements by ~2^-10 of
    absref, far above the wgmma bound of 97 accumulation steps (~2^-16)."""
    from dalle_mtf_b200 import lib as L
    from oracle import vae as OV
    g = _gen(N + H + W + Cout)
    x = torch.rand(N, H, W, 3, generator=g, device=DEV) * 2 - 1
    w = _randn(4, 4, 3, Cout, g=g, scale=0.2)
    bias = _randn(Cout, g=g, scale=0.1)
    y = nan_like((N, H // 2, W // 2, Cout), BF16)
    if kernel == "wgmma":
        ops.conv2d_first_fwd(x, w, bias, y)
        hi = x.to(BF16).float()
        lo = (x - hi).to(BF16).float()
        x_ops, w_ops, b = hi.to(F64) + lo.to(F64), w.to(BF16).to(F64), 97 * UTC
        x_abs = hi.abs().to(F64) + lo.abs().to(F64)
    else:
        L.check(L.load().db200_conv2d_first_fwd_fma(L.stream_ptr(), x.data_ptr(), w.data_ptr(), bias.data_ptr(),
                                                    y.data_ptr(), N, H, W, Cout), "conv2d_first_fwd_fma")
        x_ops, w_ops, b = x.to(F64), w.to(F64), 49 * U
        x_abs = x_ops.abs()
    ref = OV.conv2d_same(x_ops, w_ops, bias.to(F64), 2)
    absref = OV.conv2d_same(x_abs, w_ops.abs(), bias.abs().to(F64), 2)
    check(f"first layer {kernel} N={N} {H}x{W} Cout={Cout}", y, ref, absref, b=b + 4 * U, bf16_out=True)


# ------------------------------------------------------------------------------------------------------- codebook
def _bits(t):
    return t.view(torch.int16)


@pytest.mark.parametrize("n", [1_000_003, 8 * 37 + 5])
def test_split_f32_is_bit_exact(ops, n):
    g = _gen(n)
    x = torch.randn(n, generator=g, device=DEV) * torch.exp2(torch.randint(-20, 20, (n,), generator=g, device=DEV))
    bmax = torch.finfo(BF16).max
    mid = bmax + 2.0 ** 119                                 # halfway between bf16 max and the next binade (ties to inf)
    f32 = lambda v: torch.tensor(v, dtype=F32)
    special = torch.stack([
        f32(0.0), f32(-0.0), f32(1e-40), f32(-3e-42), f32(2.0 ** -149), f32(-(2.0 ** -126)), f32(1.0 + 2.0 ** -8),
        f32(1.0 + 3 * 2.0 ** -9), torch.nextafter(f32(mid), f32(0.0)), f32(mid), torch.nextafter(f32(mid), f32(math.inf)),
        f32(bmax), f32(-bmax), torch.nextafter(f32(-mid), f32(0.0)), f32(torch.finfo(F32).max), f32(1.0 / 3.0),
    ]).to(DEV)
    x[:special.numel()] = special           # vector body
    x[-special.numel():] = special          # ... and the n % 8 tail
    hi, lo = nan_like((n,), BF16), nan_like((n,), BF16)
    ops.split_f32(x, hi, lo)
    want_hi = x.to(BF16)
    want_lo = (x - want_hi.float()).to(BF16)
    assert torch.equal(_bits(hi), _bits(want_hi))
    assert torch.equal(_bits(lo), _bits(want_lo))
    print(f"[vae-kernels] split_f32 n={n}: bit-exact (worst err/bound 0)")


def _peaky_rows(rows, K, g):
    """Gumbel-softmax-like rows: softmax of logits with a spread of 3, so a few codes dominate each row."""
    return torch.softmax(torch.randn(rows, K, generator=g, device=DEV) * 3, dim=-1)


@pytest.mark.parametrize("config,B", [("vae_example_b200", 32), ("vae_coco_b200", 16)])
def test_codebook_products_of_split_operands(ops, config, B):
    """VaeEngine's codebook products on wgmma in bf16 mode, through the engine's own methods: the logits, the lookup
    z = y C^T, and the quantiser backward (dy, the straight-through Gumbel gradient, the codebook gradient through
    linear_wgrad with automatic split-K, denc).  Compared with float64 products of the unsplit fp32 operands, within
    the split bound (SPLIT1 / SPLIT2 above) plus the accumulation bound of their contraction length."""
    eng = _engine(config)
    assert eng._cb_tc
    n_hid, K = eng.n_hid, eng.K
    rows = B * eng.image_seq_len
    g = _gen(rows + K)
    C = eng.P("codebook/codebook")
    C.copy_(torch.rand(n_hid, K, generator=g, device=DEV) * 2 - 1)
    eng.refresh_shadow()
    eng._alloc(B)
    b = eng._b
    C64 = C.to(F64)

    def mm(a, bb):
        return a.to(F64) @ bb.to(F64), a.abs().to(F64) @ bb.abs().to(F64)

    # logits = x @ (C_hi + C_lo), x exactly bf16 (the last encoder activation)
    xb = _randn(rows, n_hid, g=g, dtype=BF16)
    b["logits"].fill_(NAN)
    logits = eng._codebook_logits(xb, rows)
    ref, absref = mm(xb, C64)
    check(f"{config} logits rows={rows}", logits, ref, absref, b=SPLIT1 + (n_hid + 8) * UTC)
    del ref, absref
    # z = y @ C^T through the engine's codebook lookup (splits y_out, three products); soft Gumbel: y_out = y_soft
    y = _peaky_rows(rows, K, g)
    b["y_out"].copy_(y)
    b["y_soft"].copy_(y)
    b["z_f32"].fill_(NAN)
    eng._codebook_lookup(B)
    ref, absref = mm(y, C64.t())
    check(f"{config} z = y C^T rows={rows}", b["z_f32"], ref, absref, b=SPLIT2 + (K + 8) * UTC)
    del ref, absref
    # quantiser backward for dz = d(loss)/dz (bf16, the decoder's input gradient), codebook gradient onto a base
    tau = 0.5
    eng._tau = tau
    dzb = _randn(rows, n_hid, g=g, scale=1e-3, dtype=BF16)
    base = torch.randn(n_hid, K, generator=g, device=DEV) * 0.1
    gcb = eng.G("codebook/codebook")
    gcb.copy_(base)
    for name in ("dy", "dlogits", "denc_f32"):
        b[name].fill_(NAN)
    eng._quantiser_backward(dzb, rows)
    ref, absref = mm(dzb, C64)
    check(f"{config} dy = dz C rows={rows}", b["dy"], ref, absref, b=SPLIT1 + (n_hid + 8) * UTC)
    del ref, absref
    y64, dy64 = y.to(F64), b["dy"].to(F64)        # the Gumbel backward of the dy the engine computed
    ref = y64 * (dy64 - (y64 * dy64).sum(-1, keepdim=True)) / tau
    absref = y64 * (dy64.abs() + (y64 * dy64).abs().sum(-1, keepdim=True)) / tau
    check(f"{config} dlogits rows={rows}", b["dlogits"], ref, absref, a=4 * U, b=(K / 32 + 8) * U,
          floor=2.0 ** -149 / tau)
    del ref, absref, y64, dy64
    dl = b["dlogits"]                               # split into hi + lo by the engine before both products
    ref, absref = mm(dl, C64.t())
    check(f"{config} denc = dl C^T rows={rows}", b["denc_f32"], ref, absref, b=SPLIT2 + (K + 8) * UTC)
    del ref, absref
    r1, a1 = mm(dzb.t(), y)
    r2, a2 = mm(xb.t(), dl)
    check(f"{config} codebook grad rows={rows}", gcb, base.to(F64) + r1 + r2, base.abs().to(F64) + a1 + a2,
          b=SPLIT1 + (rows + 64) * UTC)


# ------------------------------------------------------------------------------------------------------- rowmatmul
@pytest.mark.parametrize("rows,K,N", [(8192, 256, 512), (8192, 512, 256), (1000, 100, 70), (1000, 70, 100)])
@pytest.mark.parametrize("b_transposed", [False, True])
@pytest.mark.parametrize("accumulate", [0, 1])
def test_rowmatmul(ops, rows, K, N, b_transposed, accumulate):
    """out = [out +] a @ b (b stored [K][N], or [N][K] when transposed): the fp32 engine's codebook products
    (vae_example: n_hid 256, K 512) and ragged sizes."""
    g = _gen(rows + K + N)
    a = torch.randn(rows, K, generator=g, device=DEV)
    bm = torch.randn(N, K, generator=g, device=DEV) if b_transposed else torch.randn(K, N, generator=g, device=DEV)
    base = torch.randn(rows, N, generator=g, device=DEV) * 4
    out = base.clone() if accumulate else nan_like((rows, N), F32)
    ops.rowmatmul(a, bm, out, rows, K, N, b_transposed=b_transposed, accumulate=bool(accumulate))
    b64 = bm.to(F64).t() if b_transposed else bm.to(F64)
    ref = a.to(F64) @ b64
    absref = a.abs().to(F64) @ b64.abs()
    if accumulate:
        ref, absref = ref + base.to(F64), absref + base.abs().to(F64)
    check(f"rowmatmul {rows}x{K}x{N} bT={int(b_transposed)} acc={accumulate}", out, ref, absref,
          b=6 * (K + 8) * UTC)


@pytest.mark.parametrize("rows,M,N", [(8192, 256, 512), (1000, 100, 70)])
def test_rowmatmul_tn_accumulates(ops, rows, M, N):
    """out[M][N] += a^T b: the fp32 engine's codebook gradient, onto a non-zero base."""
    g = _gen(rows + M + N)
    a = torch.randn(rows, M, generator=g, device=DEV)
    bm = torch.randn(rows, N, generator=g, device=DEV)
    base = torch.randn(M, N, generator=g, device=DEV) * 30
    out = base.clone()
    ops.rowmatmul_tn(a, bm, out, rows, M, N)
    ref = base.to(F64) + a.to(F64).t() @ bm.to(F64)
    absref = base.abs().to(F64) + a.abs().to(F64).t() @ bm.abs().to(F64)
    check(f"rowmatmul_tn {rows}x{M}x{N}", out, ref, absref, b=6 * (rows + 64) * UTC)


# ------------------------------------------------------------------------------------------------------- Gumbel
def _uniform_noise(rows, K, g):
    u = (torch.rand(rows, K, generator=g, device=DEV) * (1 - 1e-9) + 1e-9).clamp_(1e-9, 1 - 2.0 ** -24)
    u[:, 0] = 1e-9                          # both ends of [1e-9, 1)
    u[:, -1] = 1 - 2.0 ** -24
    return u


def gumbel_ref(logits, u, tau):
    """float64 softmax((l - log(-log u)) / tau) of the fp32 inputs and the per-element bound of the fp32 kernel."""
    l64 = logits.to(F64)
    g64 = -torch.log(-torch.log(u.to(F64))) if u is not None else torch.zeros_like(l64)
    z = (l64 + g64) / tau
    zm = z.max(-1, keepdim=True).values
    y = torch.softmax(z, dim=-1)
    dz = 2.0 ** -21 * (1 + l64.abs() + g64.abs()) / tau + U * (z - zm).abs()
    K = logits.shape[-1]
    rel = dz + 2 * dz.max(-1, keepdim=True).values + 2.0 ** -20 + (K / 32 + 8) * U
    return y, 1.1 * y * rel + 2.0 ** -148


@pytest.mark.parametrize("K,rows", [(512, 4096), (8192, 512), (100, 3001)])
@pytest.mark.parametrize("hard", [True, False])
def test_gumbel_softmax_forward(ops, K, rows, hard):
    g = _gen(K + rows + hard)
    logits = torch.randn(rows, K, generator=g, device=DEV) * 2
    for tau in (1.0, 0.5, 1.0 / 16):
        for noise in (False, True):
            u = _uniform_noise(rows, K, g) if noise else None
            y_soft, y_out = nan_like((rows, K), F32), nan_like((rows, K), F32)
            idx = torch.full((rows,), -1, dtype=I32, device=DEV)
            ops.gumbel_softmax_fwd(logits, u, y_soft, y_out, idx, rows, K, tau, hard)
            ref, bound = gumbel_ref(logits, u, tau)
            name = f"gumbel fwd K={K} tau={tau:g} u={'U[1e-9,1)' if noise else 'None'} hard={int(hard)}"
            check(name, y_soft, ref, bound, a=0.0, b=1.0)
            # idx is the first maximum of the y the kernel wrote (tf.argmax(y)), and one of the reference's maxima
            assert torch.equal(idx.long(), first_argmax(y_soft)), name
            best = ref.gather(1, idx.long()[:, None])[:, 0]
            assert (best >= ref.max(-1).values - 2 * bound.max(-1).values).all(), name
            if hard:
                assert torch.equal(y_out, torch.nn.functional.one_hot(idx.long(), K).float()), name
            else:
                assert torch.equal(y_out, y_soft), name


def test_gumbel_softmax_ties_take_the_first_maximum_of_y(ops):
    """Exact ties (neighbours, the same lane k / k + 32, an all-equal row) and near ties: z's one ulp apart round to
    the same y = 1 / sum, and then tf.argmax(y) takes the lower index although the later z is larger."""
    K = 512
    rows = []
    g = _gen(7)
    base = lambda: torch.rand(K, generator=g, device=DEV) * -3 - 1           # everything else well below
    a = torch.tensor(0.1, dtype=F32, device=DEV)
    a_up = torch.nextafter(a, torch.tensor(1.0, device=DEV))
    want = []
    for i, j in ((5, 6), (7, 39), (100, 101), (31, 32)):                      # exact ties
        r = base(); r[i] = r[j] = 3.0; rows.append(r); want.append(i)
    rows.append(torch.full((K,), 0.25, device=DEV)); want.append(0)           # all equal
    for i, j in ((9, 41), (9, 40), (9, 10), (200, 511)):                      # near ties, larger z later
        r = base(); r[i] = a; r[j] = a_up; rows.append(r); want.append(i)
    logits = torch.stack(rows).contiguous()
    n = logits.shape[0]
    for hard in (True, False):
        y_soft, y_out = nan_like((n, K), F32), nan_like((n, K), F32)
        idx = torch.full((n,), -1, dtype=I32, device=DEV)
        ops.gumbel_softmax_fwd(logits, None, y_soft, y_out, idx, n, K, 1.0, hard)
        assert torch.equal(idx.long(), first_argmax(y_soft)), (idx.tolist(), first_argmax(y_soft).tolist())
        assert idx.tolist() == want
        if hard:
            assert torch.equal(y_out, torch.nn.functional.one_hot(idx.long(), K).float())
        else:
            assert torch.equal(y_out, y_soft)
    print("[vae-kernels] gumbel ties / near ties: idx = first maximum of y_soft (worst err/bound 0)")


def test_gumbel_softmax_non_finite_rows_stay_in_their_row(ops):
    """A NaN or +inf logit, or a row of -inf, makes every y of the row NaN: no y is a maximum.  The hard forward must
    still give an index in [0, K) (the kernel's choice is 0) and write only its own row of y_out; the finite rows are
    unaffected.  y_out is a slice of a larger buffer whose guard rows must stay untouched."""
    K, rows = 512, 8
    g = _gen(11)
    logits = torch.randn(rows, K, generator=g, device=DEV)
    logits[1, 17] = NAN
    logits[3, 200] = math.inf
    logits[5] = -math.inf
    logits[6, 3] = NAN
    logits[6, 300] = math.inf
    bad = torch.tensor([1, 3, 5, 6], device=DEV)
    good = torch.tensor([0, 2, 4, 7], device=DEV)
    buf = torch.full((rows + 2, K), -7.0, device=DEV)
    y_out = buf[1:-1]
    y_soft = nan_like((rows, K), F32)
    idx = torch.full((rows,), -1, dtype=I32, device=DEV)
    ops.gumbel_softmax_fwd(logits, None, y_soft, y_out, idx, rows, K, 1.0, True)
    torch.cuda.synchronize()
    assert ((idx >= 0) & (idx < K)).all(), idx.tolist()
    assert (idx[bad] == 0).all(), idx.tolist()
    assert torch.isnan(y_soft[bad]).all()
    assert (buf[0] == -7.0).all() and (buf[-1] == -7.0).all()
    assert torch.equal(y_out, torch.nn.functional.one_hot(idx.long(), K).float())
    assert torch.equal(idx[good].long(), first_argmax(y_soft[good]))
    print("[vae-kernels] gumbel non-finite rows: idx 0, writes stay in the row (worst err/bound 0)")


@pytest.mark.parametrize("K,rows", [(512, 4096), (8192, 512), (100, 3001)])
@pytest.mark.parametrize("tau", [1.0, 1.0 / 16])
def test_gumbel_softmax_backward(ops, K, rows, tau):
    """dlogits = y (dy - sum(y dy)) / tau for the kernel's own y_soft."""
    g = _gen(K * 3 + rows)
    logits = torch.randn(rows, K, generator=g, device=DEV) * 2
    y = nan_like((rows, K), F32)
    ops.gumbel_softmax_fwd(logits, None, y, None, None, rows, K, tau, False)
    dy = torch.randn(rows, K, generator=g, device=DEV)
    dl = nan_like((rows, K), F32)
    ops.gumbel_softmax_bwd(y, dy, dl, rows, K, tau)
    y64, d64 = y.to(F64), dy.to(F64)
    dot = (y64 * d64).sum(-1, keepdim=True)
    ref = y64 * (d64 - dot) / tau
    absref = y64.abs() * (d64.abs() + (y64 * d64).abs().sum(-1, keepdim=True)) / tau
    # y * (d - dot) rounds in the subnormal range for y near underflow (<= 2^-150 absolute), then is scaled by 1/tau
    check(f"gumbel bwd K={K} tau={tau:g}", dl, ref, absref, a=4 * U, b=(K / 32 + 8) * U, floor=2.0 ** -149 / tau)


# ------------------------------------------------------------------------------------------------------- argmax
@pytest.mark.parametrize("K", [512, 8192, 100, 33])
def test_argmax_rows_first_maximum(ops, K):
    g = _gen(K)
    rows = 2000
    x = torch.randn(rows, K, generator=g, device=DEV)
    r = torch.arange(rows, device=DEV)
    i = torch.randint(0, K, (rows,), generator=g, device=DEV)
    x[r[:500], i[:500]] = 10.0
    x[r[:250], ((i[:250] + 1) % K)] = 10.0                     # ties across lanes (neighbours)
    x[r[250:500], ((i[250:500] + 32) % K)] = 10.0              # ties within a lane (k, k + 32; wraps for K < 64)
    x[500:700] = 1.5                                           # all equal
    x[700:900, ::3] = -math.inf                                # -inf entries
    x[900:910] = -math.inf                                     # all -inf
    x[910:1000] = torch.randint(-2, 3, (90, K), generator=g, device=DEV).float()   # many ties
    idx = torch.full((rows,), -1, dtype=I32, device=DEV)
    ops.argmax_rows(x, idx, rows, K)
    assert torch.equal(idx.long(), first_argmax(x))
    # a row of NaN has no maximum: the token id must still be a valid one (0)
    nan_rows = torch.full((5, K), NAN, device=DEV)
    nidx = torch.full((5,), -1, dtype=I32, device=DEV)
    ops.argmax_rows(nan_rows, nidx, 5, K)
    assert (nidx == 0).all(), nidx.tolist()
    print(f"[vae-kernels] argmax_rows K={K}: first maximum everywhere (worst err/bound 0)")


# ------------------------------------------------------------------------------------------------------- mse
@pytest.mark.parametrize("n", [32 * 256 * 256 * 3, 1_000_003])
def test_mse_loss_and_gradient(ops, n):
    g = _gen(n)
    p = torch.randn(n, generator=g, device=DEV)
    t = torch.rand(n, generator=g, device=DEV) * 2 - 1
    scale = 1.0 / n
    dp = nan_like((n,), F32)
    acc = torch.full((1,), 0.75, device=DEV)
    ops.mse_fwd_bwd(p, t, dp, acc, scale)
    s32 = torch.tensor(scale, dtype=F32, device=DEV)
    assert torch.equal(dp, 2 * (p - t) * s32)                          # bit-equal to fp32 2 (p - t) scale
    ref = 0.75 + float(s32) * ((p.to(F64) - t.to(F64)) ** 2).sum()
    grid = min(-(-n // 256), 8 * _sm())
    depth = -(-n // (grid * 256)) + 5 + 8 + grid                       # thread chain, warp, block, atomics
    check(f"mse n={n}", acc, ref.reshape(1), ref.reshape(1), a=0.0, b=(depth + 8) * U)


# ------------------------------------------------------------------------------------------------------- s2d
@pytest.mark.parametrize("s,C", [(2, 3), (4, 3), (2, 5)])
def test_space_to_depth_is_bit_exact(ops, s, C):
    from oracle import vae as OV
    g = _gen(s * 10 + C)
    N, H, W = 3, 24, 40
    x = torch.randn(N, H, W, C, generator=g, device=DEV)
    deep = nan_like((N, H // s, W // s, C * s * s), F32)
    ops.space_to_depth(x, deep, s)
    assert torch.equal(deep, OV.space_to_depth(x, s))
    d2 = torch.randn(N, H // s, W // s, C * s * s, generator=g, device=DEV)
    flat = nan_like((N, H, W, C), F32)
    ops.space_to_depth(d2, flat, s, inverse=True)
    assert torch.equal(flat, OV.depth_to_space(d2, s))
    back = nan_like((N, H, W, C), F32)
    ops.space_to_depth(deep, back, s, inverse=True)
    assert torch.equal(back, x)
    print(f"[vae-kernels] space_to_depth s={s} C={C}: bit-exact both ways (worst err/bound 0)")


# ------------------------------------------------------------------------------------------------------- determinism
def test_bench_tokenizer_tokens_are_bitwise_reproducible():
    """encode_tokens at the bench tokenizer's batch: the forward convolutions, the split, the codebook product and the
    argmax use no atomics, so two calls give identical token ids (bench.py --dump-outputs compares them)."""
    cfg = _config("vae_example_b200")
    eng = _engine("vae_example_b200")
    eng.init_params(seed=3)
    g = _gen(3)
    B, size = cfg["train_batch_size"], cfg["dataset"]["image_size"]
    img = torch.rand(B, size, size, 3, generator=g, device=DEV) * 2 - 1
    t1 = eng.encode_tokens(img).clone()
    t2 = eng.encode_tokens(img).clone()
    assert t1.shape == (B, eng.image_seq_len)
    assert torch.equal(t1, t2)
    assert int(t1.min()) >= 0 and int(t1.max()) < eng.K and t1.unique().numel() > 1
    print(f"[vae-kernels] encode_tokens B={B}: bitwise identical twice (worst err/bound 0)")
