"""The DALL-E paper's discrete-VAE network (PaperVaeEngine) against float64, per element, at the shapes its engine
launches: the block convolutions (1x1 and 3x3, wgmma and direct), the 7x7 input conv, pool, upsample, residual_gain,
the casts, and the two f32 projections as bf16 hi + lo products with a bias.

The conventions are those of test_vae_kernels_gpu.py (imported as VK, whose run_conv and bounds this module reuses):
the kernel and the float64 reference read the same operands, outputs start as NaN, outputs a kernel accumulates into
start from a non-zero base, and each element must satisfy |got - ref| <= a |ref| + b absref (bf16 outputs: half a
bf16 ulp at |ref| instead of a |ref|).  One `[vae-paper-kernels] ...: worst err/bound r` line per case.

  1. A recorder wraps the ops functions and notes every distinct launch at the outermost ops call (linear_wgrad, not
     the gemm inside it): its entry point, descriptor and which of bias / mask / residual it passes, and whether the
     residual gradient is the output buffer.  It runs at the vae_paper_b200 geometry (256^2, n_hid 256, 2 blocks x 4
     groups, n_init 128, K 8192, bf16, logit-Laplace, KL on, soft Gumbel): one training step at 8 images per GPU
     (64 over data:8), encode_tokens at 16 (dalle_coco_paper_vae_b200 tokenises 128 over data:8) and decode_tokens at
     dalle_coco_paper_vae_b200's predict_batch_size, the images generate_dalle.py decodes in one call (the engine
     runs them in passes of at most decode_pass_images()).
  2. Every recorded launch class is replayed at its recorded batch (convolutions through VK.run_conv with exactly the
     recorded flag sets), checked on the engine's own operands (the projections), or named in EXEMPT with the test
     that pins its class at equal or larger size.  Anything else fails test_every_recorded_launch_is_checked.
  3. The projections are checked on the buffers the engine keeps after one bf16 step; the projection weights are drawn
     positive with a lo part of 0.4 bf16 ulp, so that dropping a lo product moves the outputs above the bound.
  4. One bf16 step at 2 images checks every convolution launch on exactly the operands it read (post-ReLU sparsity,
     1/64-gain residuals, bf16 ties), the residual gradient cloned before it is overwritten in place.
  5. The f32 engine's convolutions at the four small geometries of test_vae_paper_gpu.py, and the B = 8 bf16 classes
     again with 4 SMs reserved (the data-parallel overlap window, where the wgrad pixel splits change).
Each check also runs a mutated reference that must fail: the mask or the residual gradient dropped, a 1x1 output one
pixel over, a projection without its lo part, the bias added twice, a weight gradient without its base.

On an H100 80GB HBM3 (132 SMs, 700 W power limit) the module takes 30 s (pytest's count), the float64 replays at
8 x 256^2 included.
"""
import functools
import math

import pytest
import torch

import float64_bounds
import test_vae_kernels_gpu as VK
import test_vae_paper_gpu as VP
from float64_bounds import DEV, U, UTC, nan_like
from launch_census import OpsRecorder

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
TAG = "vae-paper-kernels"
check = functools.partial(float64_bounds.check, tag=TAG)
must_fail = VK.must_fail

PAPER = dict(n_hid=256, n_blk_per_group=2, group_count=4, n_init=128)
K_PAPER, SIZE = 8192, 256
TRAIN_B, TOKENIZE_B = 8, 16          # vae_paper_b200: 64 over data:8; dalle_coco_paper_vae_b200: 128 over data:8
DECODE_B = VK._config("dalle_coco_paper_vae_b200")["predict_batch_size"]
TAU, BETA = 0.7, 0.034375

CONV_ENTRIES = ("conv2d_fwd", "conv2d_fwd_tc", "conv2d_dgrad", "conv2d_dgrad_tc", "conv2d_wgrad", "conv2d_wgrad_tc")
BIT_EXACT = ("cast_f32_to_bf16", "cast_bf16_to_f32", "split_f32", "onehot_rows", "argmax_rows")
K11P = ("conv7x7_in_fwd", "conv7x7_in_wgrad", "maxpool2x2_fwd", "maxpool2x2_bwd", "upsample2x_fwd", "upsample2x_bwd",
        "residual_gain")
PROJECTION = ("gemm", "linear_wgrad", "colsum")
HOST_ONLY = ("conv_desc", "conv_tc_supported", "conv_dgrad_tc_supported", "conv_wgrad_tc_supported")   # no launch
# entry point -> the test of this module that checks every recorded class of it
CHECKED = {**{e: "test_block_convolutions_at_the_recorded_batch" for e in CONV_ENTRIES},
           **{e: "test_k11p_kernels_at_the_recorded_sizes" for e in K11P},
           **{e: "test_casts_one_hot_and_argmax_at_the_recorded_sizes" for e in BIT_EXACT},
           **{e: "test_projections_on_the_engine_operands" for e in PROJECTION}}
# entry point -> (test that pins its class, why that size covers the recorded one)
EXEMPT = {
    "gumbel_softmax_fwd": ("test_vae_kernels_gpu.py::test_gumbel_softmax_forward[*-8192-512]",
                           "row-local softmax: K = 8192 is pinned per element, soft and hard, noise and no noise; "
                           "rows are independent CTAs, so 8192 rows add no other arithmetic"),
    "gumbel_softmax_bwd_kl": ("test_vae_kl_gpu.py::test_kl_backward_against_float64[16384-8192-2.0]",
                              "K = 8192 at 16384 rows, twice the recorded 8192"),
    "vae_kl_stats": ("test_vae_kl_gpu.py::test_kl_stats_against_float64[16384-8192]",
                     "K = 8192 at 16384 rows, twice the recorded 8192"),
    "logit_laplace": ("test_vae_logit_laplace_gpu.py::test_logit_laplace_kernel_against_float64[1048576-3] and "
                      "test_logit_laplace_decode_mode_writes_only_the_image[1048576-3]",
                      "16 x 256^2 pixels of 3 channels (the vae_coco rows), the recorded training step's 8 x 256^2 "
                      "and the decode passes of at most 16 x 256^2"),
}


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------------- recorder
class Launch:
    """One launch: entry point, hashable class key, role (fwd / dgrad / wgrad / None) and the parameter whose weight
    or weight gradient it reads or writes (None for the rest)."""

    def __init__(self, entry, key, role=None, weight=None, geo=None, flags=None):
        self.entry, self.key, self.role, self.weight, self.geo, self.flags = entry, key, role, weight, geo, flags or {}


def _tensor_sig(v):
    if isinstance(v, torch.Tensor):
        return (tuple(v.shape), str(v.dtype))
    if isinstance(v, (int, float, bool)) or v is None:
        return v
    return type(v).__name__


def _same(a, b):
    return isinstance(a, torch.Tensor) and isinstance(b, torch.Tensor) and a.data_ptr() == b.data_ptr()


def describe(entry, A, names):
    """Launch of `entry` called with the bound arguments A; names maps weight data pointers to parameter names."""
    wname = lambda t: names.get(t.data_ptr()) if isinstance(t, torch.Tensor) else None
    if entry in CONV_ENTRIES:
        c = A["c"]
        geo = (c.N, c.H, c.W, c.Cin, c.Cout, c.KH, c.KW, c.stride, bool(c.transposed), bool(c.act_f32))
        if "fwd" in entry:
            role, w = "fwd", A.get("w", A.get("w_bf16"))
            flags = dict(relu=bool(c.relu), bias=A["bias"] is not None, residual=A["residual"] is not None)
        elif "dgrad" in entry:
            role, w = "dgrad", A.get("w", A.get("w_bf16"))
            flags = dict(mask=A["x_mask"] is not None, dres=A["dres"] is not None, in_place=_same(A["dres"], A["dx"]))
        else:
            role, w = "wgrad", A["dw"]
            flags = dict(dbias=A.get("dbias") is not None)
        return Launch(entry, (entry, geo, tuple(sorted(flags.items()))), role, wname(w), geo, flags)
    if entry == "gemm":
        key = (entry, A["M"], A["N"], A["K"], A["a_mn"], A["b_mn"], A["mode"], A["bias"] is not None, A["split_k"])
        return Launch(entry, key, "fwd" if A["b_mn"] else "dgrad", wname(A["b"]))
    if entry == "linear_wgrad":
        return Launch(entry, (entry, tuple(A["x"].shape), tuple(A["dy"].shape)), "wgrad", wname(A["dw"]))
    if entry == "conv7x7_in_fwd":
        return Launch(entry, (entry, _tensor_sig(A["x_f32"]), _tensor_sig(A["y"])), "fwd", wname(A["w"]))
    if entry == "conv7x7_in_wgrad":
        return Launch(entry, (entry, _tensor_sig(A["x_f32"]), _tensor_sig(A["dy"]), A["dbias"] is not None), "wgrad",
                      wname(A["dw"]))
    if entry == "residual_gain":
        flags = dict(gain=float(A["gain"]), id=A["id"] is not None, mask=A["mask"] is not None,
                     y=A["y"] is not None, relu_y=A["relu_y"] is not None, in_place=_same(A["y"], A["r"]))
        return Launch(entry, (entry, _tensor_sig(A["r"]), tuple(sorted(flags.items()))), flags=flags)
    return Launch(entry, (entry,) + tuple(_tensor_sig(v) for v in A.values()))


def weight_names(eng):
    """data pointer -> parameter name (without /kernel) of every kernel's master, gradient and bf16 copies."""
    names = {}
    for name in eng.layout.order:
        if name.endswith("/kernel"):
            base = name[:-len("/kernel")]
            names[eng.P(name).data_ptr()] = names[eng.G(name).data_ptr()] = base
            if eng.shadow is not None:
                names[eng.W16(name).data_ptr()] = base
    if eng.use_bf16:
        for t in (eng.eo_hi, eng.eo_lo):
            names[t.data_ptr()] = "encoder/output/conv"
        for t in (eng.di_hi, eng.di_lo):
            names[t.data_ptr()] = "decoder/input"
    return names


class Recorder(OpsRecorder):
    """OpsRecorder of the outermost ops calls (a wrapper calling another, as linear_wgrad calls gemm, counts once),
    each described as a Launch with the engine's weight names."""

    def __init__(self, eng, before=None, after=None):
        self.names = weight_names(eng)
        super().__init__(lambda entry, A: (describe(entry, A, self.names), None), skip=HOST_ONLY, before=before,
                         after=after)


def distinct(launches):
    seen = {}
    for l in launches:
        seen.setdefault(l.key, l)
    return list(seen.values())


# ------------------------------------------------------------------------------------------------------- the engine
def split_heavy(shape, g, std):
    """Positive f32 weights whose bf16 split has lo = 0.4 ulp of hi, with hi's sign: a product with a non-negative
    operand then loses ~2^-10 |ref| when its lo part is dropped, above the projections' bounds."""
    hi = (torch.rand(shape, generator=g, device=DEV) * std + std / 4).to(BF16).float()
    return hi + 0.4 * torch.exp2(torch.floor(torch.log2(hi)) - 7)


def paper_engine(seed=0, heavy_lo=True):
    """The vae_paper_b200 network with its own initialisation and biases of std 0.1; heavy_lo: the projection
    weights from split_heavy (positive, so the decoder input z > 0 almost everywhere: the real-operand test keeps the
    signed initial weights, under which the first decoder block's ReLU mask drops half of z)."""
    from dalle_mtf_b200.vae_paper_engine import PaperVaeEngine
    eng = PaperVaeEngine(K_PAPER, SIZE, use_bf16=True, kl=True, reconstruction_loss="logit_laplace", **PAPER)
    eng.init_params(seed)
    g = _gen(seed + 1)
    for name in eng.layout.order:
        if name.endswith("/bias"):
            eng.P(name).copy_(torch.randn(eng.P(name).shape, generator=g, device=DEV) * 0.1)
    if heavy_lo:
        eng.P("encoder/output/conv/kernel").copy_(split_heavy((1, 1, eng.n_hid, eng.K), g, 2.0 / eng.n_hid))
        eng.P("decoder/input/kernel").copy_(split_heavy((1, 1, eng.K, eng.n_init), g, 2.0))
    eng.refresh_shadow()
    assert torch.equal(eng.eo_hi.float(), eng.P("encoder/output/conv/kernel").view(eng.n_hid, eng.K).to(BF16).float())
    return eng


def step_inputs(eng, B, seed):
    g = _gen(seed)
    img = torch.rand(B, SIZE, SIZE, 3, generator=g, device=DEV) * 2 - 1
    u = (torch.rand(B * eng.image_seq_len, eng.K, generator=g, device=DEV)).clamp_(1e-9, 1 - 2.0 ** -24)
    return img, u


def train_step(eng, img, u, seed_grads=None):
    eng.zero_grads()
    eng.forward(img, u, TAU, False, kl_weight=BETA)
    if seed_grads:
        for name, t in seed_grads.items():
            eng.G(name).copy_(t.view(eng.G(name).shape))
    eng.backward()


PROJ_PARAMS = ("encoder/output/conv/kernel", "encoder/output/conv/bias", "decoder/input/kernel", "decoder/input/bias")


@pytest.fixture(scope="module")
def paper_run(ops):
    """Launches of the vae_paper_b200 step at B = 8, of encode_tokens at B = 16 and of decode_tokens at DECODE_B, and
    the B = 8 step's projection operands and results (a second step with the projection gradients seeded with bases
    sized from the first)."""
    eng = paper_engine()
    img, u = step_inputs(eng, TRAIN_B, 1)
    cap = {}

    def after(entry, A, _):
        b = eng._b
        if entry == "linear_wgrad" and _same(A["x"], b.get("y_hi")):
            cap["dz"] = A["dy"].clone()
        if entry == "residual_gain" and A["mask"] is not None and _same(A["y"], A["r"]):
            cap["relu_bwd"] = A["y"].clone()
            cap["enc_last"] = A["mask"].clone()

    with Recorder(eng, after=after) as rec:
        train_step(eng, img, u)
        torch.cuda.synchronize()
    train_launches = list(rec.launches)
    # bases for the projection gradients: larger than their bound, so that a kernel that drops one fails
    b = eng._b
    rows = TRAIN_B * eng.image_seq_len
    a = b["enc_relu"].view(rows, eng.n_hid).to(F64).abs()
    abs_e = a.t() @ b["dlogits"].to(F64).abs()
    abs_d = b["y_out"].to(F64).abs().t() @ cap["dz"].to(F64).abs()
    del a
    g = _gen(5)
    bases = {}
    for name, absref, L in (("encoder/output/conv/kernel", abs_e, rows), ("decoder/input/kernel", abs_d, rows)):
        bw = VK.SPLIT1 + (L + 64) * UTC
        bases[name] = torch.randn(absref.shape, generator=g, device=DEV) * (4 * bw * float(absref.max()) / (1 - bw))
        bases[name.replace("kernel", "bias")] = torch.randn(absref.shape[1], generator=g, device=DEV)
    del abs_e, abs_d
    with Recorder(eng, after=after):
        train_step(eng, img, u, seed_grads=bases)
        torch.cuda.synchronize()
    keep = {k: b[k].clone() for k in ("enc_relu", "logits", "y_out", "z_f32", "dy", "dlogits", "denc_f32")}
    keep.update(cap)
    keep.update({"grad/" + n: eng.G(n).clone() for n in PROJ_PARAMS})
    keep.update({"param/" + n: eng.P(n).clone() for n in PROJ_PARAMS})
    keep["bases"] = bases
    keep["hw"], keep["n_hid"], keep["n_init"] = eng.hw, eng.n_hid, eng.n_init
    # the tokenizer's launches at 16 images, decoding at DECODE_B
    img16, _ = step_inputs(eng, TOKENIZE_B, 2)
    with Recorder(eng) as rec:
        tokens = eng.encode_tokens(img16).clone()
        codes = tokens.repeat(_cdiv(DECODE_B, TOKENIZE_B), 1)[:DECODE_B].contiguous()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        held = torch.cuda.memory_allocated()
        images = eng.decode_tokens(codes)
        torch.cuda.synchronize()
    assert images.shape == (DECODE_B, SIZE, SIZE, 3) and torch.isfinite(images).all()
    print(f"[{TAG}] decode_tokens B={DECODE_B} in passes of {eng.decode_pass_images()}: peak allocation "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB, {held / 2 ** 30:.1f} GiB of it held before the call "
          f"(the engine with its 16-image tokenizer buffers, which the first pass replaces)")
    del images, codes
    token_launches = list(rec.launches)
    del eng
    torch.cuda.empty_cache()
    return {"train": train_launches, "tokens": token_launches, "all": train_launches + token_launches, "step": keep}


# ------------------------------------------------------------------------------------------------------- coverage
def test_recorded_launches_name_every_kernel_of_the_network(paper_run):
    """Every kernel of oracle.vae_paper.param_shapes has a forward and a weight-gradient launch, and a dgrad launch
    unless it is encoder/input (the image needs no gradient)."""
    from oracle import vae_paper as OP
    roles = {}
    for l in paper_run["train"]:
        if l.role:
            assert l.weight is not None, (l.entry, l.key)
            roles.setdefault(l.weight, set()).add(l.role)
    want = [n[:-len("/kernel")] for n in OP.param_shapes(K_PAPER, **PAPER) if n.endswith("/kernel")]
    assert sorted(roles) == sorted(want)
    for n in want:
        assert roles[n] == ({"fwd", "wgrad"} if n == "encoder/input" else {"fwd", "dgrad", "wgrad"}), (n, roles[n])
    convs = [l for l in distinct(paper_run["train"]) if l.entry in CONV_ENTRIES]
    # the paper's block shapes: 1x1 convs, and the mask + in-place residual gradient in one dgrad
    assert any(l.geo[5] == 1 and l.entry == "conv2d_fwd_tc" for l in convs)
    assert any(l.flags.get("mask") and l.flags.get("in_place") for l in convs)
    print(f"[{TAG}] recorded: {len(distinct(paper_run['all']))} launch classes, {len(want)} kernels "
          f"(worst err/bound 0)")


def test_every_recorded_launch_is_checked(paper_run):
    """A recorded entry point is checked by a test of this module or pinned elsewhere (EXEMPT); an exemption for an
    entry point that no longer runs is stale."""
    entries = {l.entry for l in paper_run["all"]}
    unchecked = sorted(entries - set(CHECKED) - set(EXEMPT))
    assert not unchecked, f"recorded launches that nothing here checks: {unchecked}"
    stale = sorted(set(EXEMPT) - entries)
    assert not stale, f"exemptions for entry points the engine no longer launches: {stale}"
    for l in paper_run["all"]:       # the projection test checks the products of the two projections, and only those
        if l.entry in ("gemm", "linear_wgrad"):
            assert l.weight in ("encoder/output/conv", "decoder/input"), l.key
    print(f"[{TAG}] {len(entries)} recorded entry points: {len(entries & set(CHECKED))} checked here, "
          f"{len(entries & set(EXEMPT))} pinned elsewhere (worst err/bound 0)")


# ------------------------------------------------------------------------------------------------------- convolutions
def conv_classes(ops, launches):
    """geometry (N, H, Cin, Cout, k, act_f32) -> the recorded forward and dgrad variants (VK.FWD_VARIANTS /
    DGRAD_VARIANTS) and whether a wgrad ran; checks that the engine ran the kernel run_conv picks for the shape."""
    out = {}
    for l in distinct(launches):
        if l.entry not in CONV_ENTRIES:
            continue
        N, H, W, Cin, Cout, KH, KW, stride, transposed, f32 = l.geo
        assert H == W and KH == KW and stride == 1 and not transposed, l.key
        d = out.setdefault((N, H, Cin, Cout, KH, f32), {"fwd": set(), "dgrad": set(), "wgrad": False})
        c = ops.conv_desc(N, H, W, Cin, Cout, KH, KW, 1, act_f32=f32)
        f = l.flags
        if l.role == "fwd":
            assert f["bias"] and not (f["relu"] and f["residual"]), l.key
            assert (l.entry == "conv2d_fwd_tc") == ops.conv_tc_supported(c), l.key
            d["fwd"].add("relu" if f["relu"] else "res" if f["residual"] else "plain")
        elif l.role == "dgrad":
            assert (l.entry == "conv2d_dgrad_tc") == ops.conv_dgrad_tc_supported(c), l.key
            parts = (["mask"] if f["mask"] else []) + ([("dres in place" if f["in_place"] else "dres")]
                                                       if f["dres"] else [])
            d["dgrad"].add(" ".join(parts) or "plain")
        else:
            assert (l.entry == "conv2d_wgrad_tc") == ops.conv_wgrad_tc_supported(c), l.key
            assert f["dbias"] == (l.entry == "conv2d_wgrad"), l.key     # the wgmma wgrad's bias runs on colsum
            d["wgrad"] = True
    for geo, d in out.items():      # the tokenizer's classes run forward only
        assert d["fwd"] and (d["wgrad"] or not d["dgrad"]), geo
        assert set(d["dgrad"]) <= set(VK.DGRAD_VARIANTS), (geo, d["dgrad"])
    return out


def replay_convolutions(ops, launches, label, seed=0):
    """VK.run_conv on every recorded convolution class at its recorded batch with exactly its recorded variants.
    Returns (worst ratio, [(geometry, wgrad pixel splits, pixel tiles per split)] of the wgmma wgrads)."""
    worst, splits = 0.0, []
    sm = float64_bounds.sm_count()
    for i, ((N, H, Cin, Cout, k, f32), d) in enumerate(sorted(conv_classes(ops, launches).items())):
        order = lambda s, names: tuple(v for v in names if v in s)
        tag = f"{label} {k}x{k} {Cin}->{Cout} @{H} N={N}"
        worst = max([worst] + VK.run_conv(ops, tag, N, H, Cin, Cout, k, 1, False, dgrad=bool(d["dgrad"]),
                                          wgrad=d["wgrad"], act_f32=f32, seed=seed + i,
                                          fwd_variants=order(d["fwd"], VK.FWD_VARIANTS),
                                          dgrad_variants=order(d["dgrad"], VK.DGRAD_VARIANTS), line_tag=TAG))
        c = ops.conv_desc(N, H, H, Cin, Cout, k, k, 1, act_f32=f32)
        if d["wgrad"] and ops.conv_wgrad_tc_supported(c):
            _, _, s, per = VK.wgrad_split(N, H, Cin, Cout, k, 1, False, sm)
            splits.append(((N, H, Cin, Cout, k), s, per))
    return worst, splits


def test_block_convolutions_at_the_recorded_batch(ops, paper_run):
    worst, splits = replay_convolutions(ops, paper_run["all"], "paper bf16")
    assert any(s >= 2 and per >= 2 for _, s, per in splits), splits
    print(f"[{TAG}] paper bf16 convolutions: worst err/bound {worst:.4f}")


def test_block_convolutions_with_4_sms_reserved(ops, paper_run):
    """The B = 8 classes in the data-parallel overlap window (4 SMs reserved): the wgrad pixel splits change."""
    full = float64_bounds.sm_count()
    with float64_bounds.reserved_sms(4) as sm:
        worst, splits = replay_convolutions(ops, paper_run["train"], "paper bf16", seed=500)
    changed = [g for g, s, _ in splits if VK.wgrad_split(*g[:4], g[4], 1, False, full)[2] != s]
    assert changed, splits
    print(f"[reserved-sms k=4 sm={sm}] [{TAG}] paper bf16 convolutions: worst err/bound {worst:.4f}, "
          f"{len(changed)} wgrads with other pixel splits")


@pytest.mark.parametrize("geo,K,size,B,ll,beta,hard,tau", VP.SMALL)
def test_f32_engine_convolutions_at_the_recorded_batch(ops, geo, K, size, B, ll, beta, hard, tau):
    """The f32 engine runs every convolution on the fp32 kernels, the two projections included (1x1 with Cin or
    Cout = K); n_hid 72 has an 18-channel bottleneck."""
    p, img, u, hw = VP._case(K, size, B, K + size + B, ll, geo)
    eng = VP._engine(K, size, geo, ll, beta is not None, False)
    with Recorder(eng) as rec:
        VP._engine_step(eng, p, img, u, tau, hard, beta)
    classes = conv_classes(ops, rec.launches)
    assert all(f32 for (_, _, _, _, _, f32) in classes)
    assert (B, hw, eng.n_hid, K, 1, True) in classes and (B, hw, K, geo["n_init"], 1, True) in classes
    worst, _ = replay_convolutions(ops, rec.launches, f"f32 n_hid={geo['n_hid']} K={K}", seed=900)
    print(f"[{TAG}] f32 n_hid={geo['n_hid']} K={K} {size}px B={B} convolutions: worst err/bound {worst:.4f}")


# ------------------------------------------------------------------------------------------------------- K11p
def _classes(launches, entry):
    return [l for l in distinct(launches) if l.entry == entry]


def _shape(sig):
    return sig[0]


def conv7x7_fwd_case(ops, N, H, C, Cout, dtype, seed):
    g = _gen(seed)
    x = torch.rand(N, H, H, C, generator=g, device=DEV) * 2 - 1
    w = torch.randn(7, 7, C, Cout, generator=g, device=DEV) / math.sqrt(49 * C)
    bias = torch.randn(Cout, generator=g, device=DEV) * 0.1
    y = nan_like((N, H, H, Cout), dtype)
    ops.conv7x7_in_fwd(x, w, bias, y)
    ref, mag = VP.conv7_ref(x, w, bias)
    return check(f"conv7x7_in_fwd N={N} {H}px {C}->{Cout} {dtype}", y, ref, mag, a=U, b=(49 * C + 1) * U,
                 bf16_out=dtype == BF16)


def conv7x7_wgrad_case(ops, N, H, C, Cout, dtype, seed):
    """The 7x7 weight gradient at the full recorded batch (its pixel splits depend on the pixel count)."""
    from dalle_mtf_b200 import lib as L
    g = _gen(seed)
    x = torch.rand(N, H, H, C, generator=g, device=DEV) * 2 - 1
    dy = VP.tie_tensor((N, H, H, Cout), dtype, seed)
    M = N * H * H
    xp = torch.nn.functional.pad(x.to(F64), (0, 0, 3, 3, 3, 3))
    d64 = dy.to(F64).reshape(-1, Cout)
    ref = torch.empty(7, 7, C, Cout, dtype=F64, device=DEV)
    mag = torch.empty_like(ref)
    for kh in range(7):
        for kw in range(7):
            patch = xp[:, kh:kh + H, kw:kw + H, :].reshape(-1, C)
            ref[kh, kw] = patch.t() @ d64
            mag[kh, kw] = patch.abs().t() @ d64.abs()
    del xp
    splits = L.load().db200_conv7x7_in_wgrad_workspace_bytes(N, H, H, C, Cout) // 4 // (49 * C * Cout + Cout)
    n = _cdiv(M, 4 * max(splits, 1)) + 4 + splits + 1
    b = n * U
    base_w = torch.randn(7, 7, C, Cout, generator=g, device=DEV) * max(1.0, 4 * b * float(mag.max()) / (1 - b))
    base_b = torch.randn(Cout, generator=g, device=DEV)
    dw, db = base_w.clone(), base_b.clone()
    ops.conv7x7_in_wgrad(x, dy, dw, db)
    name = f"conv7x7_in_wgrad N={N} {H}px {C}->{Cout} {dtype} splits={splits}"
    r = check(name, dw, base_w.to(F64) + ref, base_w.abs().to(F64) + mag, a=U, b=b)
    must_fail(name + " without its base", dw, ref, base_w.abs().to(F64) + mag, a=U, b=b)
    rel = ((dw.to(F64) - base_w.to(F64) - ref).norm() / ref.norm()).item()
    assert rel < VK.WGRAD_REL, (name, rel)
    sb = d64.sum(0)
    r = max(r, check(f"conv7x7_in_wgrad dbias N={N} {H}px", db, base_b.to(F64) + sb,
                     base_b.abs().to(F64) + d64.abs().sum(0), a=U, b=b))
    return r


def pool_case(ops, shape, dtype, seed):
    N, H, W, C = shape
    x = VP.tie_tensor(shape, dtype, seed)
    dy = VP.tie_tensor((N, H // 2, W // 2, C), dtype, seed + 1) + 3
    y, dx = nan_like((N, H // 2, W // 2, C), dtype), nan_like(shape, dtype)
    ops.maxpool2x2_fwd(x, y)
    ops.maxpool2x2_bwd(x, dy, dx)
    m, first = VP.pool_ref(x)
    assert torch.equal(y.to(F64), m)
    want = VP.unwindow(torch.nn.functional.one_hot(first, 4).to(F64) * dy.to(F64).unsqueeze(-1), shape)
    assert torch.equal(dx.to(F64), want)
    print(f"[{TAG}] maxpool2x2 fwd / bwd {shape} {dtype}: exact (worst err/bound 0)")


def upsample_case(ops, shape, dtype, seed, fwd=True):
    N, H, W, C = shape        # the low-resolution side
    g = _gen(seed)
    if fwd:
        x = VP.tie_tensor(shape, dtype, seed)
        y = nan_like((N, 2 * H, 2 * W, C), dtype)
        ops.upsample2x_fwd(x, y)
        assert torch.equal(y, x.repeat_interleave(2, 1).repeat_interleave(2, 2))
        print(f"[{TAG}] upsample2x fwd {shape} {dtype}: exact (worst err/bound 0)")
        return 0.0
    dy = torch.randn(N, 2 * H, 2 * W, C, generator=g, device=DEV).to(dtype)
    dx = nan_like(shape, dtype)
    ops.upsample2x_bwd(dy, dx)
    # four bf16 values of similar size add exactly in f32, so many sums land on a bf16 rounding tie, exactly half an
    # ulp away: the bound of test_vae_paper_gpu.py (2^-8 |ref| for the bf16 output) has room for that
    blocks = dy.to(F64).reshape(N, H, 2, W, 2, C)
    return check(f"upsample2x bwd {shape} {dtype}", dx, blocks.sum((2, 4)), blocks.abs().sum((2, 4)),
                 a=VP.U if dtype == BF16 else U, b=3 * U)


def residual_gain_case(ops, shape, dtype, flags, seed):
    """One recorded residual_gain variant: v = gain r (+ id), 0 where mask <= 0, into y (in place when recorded) and
    / or relu_y; rounded once in f32, then to the activation dtype."""
    r = VP.tie_tensor(shape, dtype, seed)
    idv = VP.tie_tensor(shape, dtype, seed + 1) if flags["id"] else None
    mask = VP.tie_tensor(shape, dtype, seed + 2) if flags["mask"] else None
    gain = flags["gain"]
    if flags["in_place"]:
        y = r.clone()
        rr = y
    else:
        y = nan_like(shape, dtype) if flags["y"] else None
        rr = r
    relu_y = nan_like(shape, dtype) if flags["relu_y"] else None
    ops.residual_gain(rr, gain, id=idv, mask=mask, y=y, relu_y=relu_y)
    # the engine's gains (1 and 1 / 64) are powers of two: gain r + id is exact in float64 and the kernel's fma rounds
    # it once to f32, then to the activation dtype, both to nearest even, so the output is known bit for bit
    g32 = torch.tensor(gain, dtype=F32).item()
    assert g32 == 2.0 ** round(math.log2(g32)), gain
    v = g32 * r.to(F64) + (idv.to(F64) if idv is not None else 0)
    keep = mask > 0 if mask is not None else torch.ones((), dtype=torch.bool, device=DEV)
    name = f"residual_gain {shape} {dtype} gain={gain:g}" + "".join(f" {k}" for k in ("id", "mask", "in_place")
                                                                    if flags[k])
    rounded = v.to(F32).to(dtype)
    want = torch.where(keep, rounded, torch.zeros((), dtype=dtype, device=DEV))
    if y is not None:
        assert torch.equal(y, want), name
    if relu_y is not None:
        assert torch.equal(relu_y, torch.relu(want)), name
    if mask is not None:     # mutation: the mask dropped
        assert not torch.equal(y if y is not None else relu_y, rounded if y is not None else torch.relu(rounded))
    print(f"[{TAG}] {name}: bit-exact (worst err/bound 0)")
    return 0.0


def test_k11p_kernels_at_the_recorded_sizes(ops, paper_run):
    """The 7x7 input conv (forward at 8 and 16 x 256^2, weight gradient at 8 x 256^2), pool, upsample and every
    residual_gain variant, at the recorded sizes and with the bounds of test_vae_paper_gpu.py."""
    worst = 0.0
    launches = paper_run["all"]
    for i, l in enumerate(_classes(launches, "conv7x7_in_fwd")):
        (N, H, _, C), (_, _, _, Cout) = _shape(l.key[1]), _shape(l.key[2])
        worst = max(worst, conv7x7_fwd_case(ops, N, H, C, Cout, getattr(torch, l.key[2][1].split(".")[1]), 10 + i))
    for i, l in enumerate(_classes(launches, "conv7x7_in_wgrad")):
        (N, H, _, C), (_, _, _, Cout) = _shape(l.key[1]), _shape(l.key[2])
        assert l.key[3]
        worst = max(worst, conv7x7_wgrad_case(ops, N, H, C, Cout, getattr(torch, l.key[2][1].split(".")[1]), 20 + i))
    dt = lambda sig: getattr(torch, sig[1].split(".")[1])
    for i, l in enumerate(_classes(launches, "maxpool2x2_fwd") + _classes(launches, "maxpool2x2_bwd")):
        pool_case(ops, _shape(l.key[1]), dt(l.key[1]), 30 + i)
    for i, l in enumerate(_classes(launches, "upsample2x_fwd")):
        upsample_case(ops, _shape(l.key[1]), dt(l.key[1]), 40 + i)
    for i, l in enumerate(_classes(launches, "upsample2x_bwd")):
        worst = max(worst, upsample_case(ops, _shape(l.key[2]), dt(l.key[2]), 50 + i, fwd=False))
    variants = _classes(launches, "residual_gain")
    assert any(l.flags["mask"] and l.flags["in_place"] for l in variants)
    for i, l in enumerate(variants):
        worst = max(worst, residual_gain_case(ops, _shape(l.key[1]), dt(l.key[1]), l.flags, 60 + i))
    print(f"[{TAG}] K11p at the recorded sizes: worst err/bound {worst:.4f}")


def test_casts_one_hot_and_argmax_at_the_recorded_sizes(ops, paper_run):
    """Bit-exact: f32 <-> bf16 casts (round to nearest even), the hi + lo split, the one-hot rows of decode_tokens and
    the first-maximum argmax of encode_tokens."""
    g = _gen(77)
    for l in distinct(paper_run["all"]):
        if l.entry not in BIT_EXACT:
            continue
        if l.entry in ("cast_f32_to_bf16", "split_f32"):
            (shape, _) = l.key[1]
            x = torch.randn(shape, generator=g, device=DEV) * torch.exp2(
                torch.randint(-12, 12, shape, generator=g, device=DEV).float())
            hi = nan_like(shape, BF16)
            if l.entry == "split_f32":
                lo = nan_like(shape, BF16)
                ops.split_f32(x, hi, lo)
                assert torch.equal(lo.view(torch.int16), (x - x.to(BF16).float()).to(BF16).view(torch.int16))
            else:
                ops.cast_f32_to_bf16(x, hi)
            assert torch.equal(hi.view(torch.int16), x.to(BF16).view(torch.int16)), l.key
        elif l.entry == "cast_bf16_to_f32":
            (shape, _) = l.key[1]
            x = torch.randn(shape, generator=g, device=DEV).to(BF16)
            y = nan_like(shape, F32)
            ops.cast_bf16_to_f32(x, y)
            assert torch.equal(y, x.float()), l.key
        elif l.entry == "onehot_rows":
            (rows,), _ = l.key[1]
            (_, K), _ = l.key[2]
            idx = torch.randint(0, K, (rows,), generator=g, device=DEV).to(I32)
            y = nan_like((rows, K), F32)
            ops.onehot_rows(idx, y)
            assert torch.equal(y, torch.nn.functional.one_hot(idx.long(), K).float()), l.key
        else:   # argmax_rows
            (rows, K), _ = l.key[1]
            x = torch.randint(-3, 4, (rows, K), generator=g, device=DEV).float()      # many ties
            idx = torch.full((rows,), -1, dtype=I32, device=DEV)
            ops.argmax_rows(x, idx, rows, K)
            assert torch.equal(idx.long(), VK.first_argmax(x)), l.key
        print(f"[{TAG}] {l.entry} {l.key[1]}: bit-exact (worst err/bound 0)")


# ------------------------------------------------------------------------------------------------------- projections
def _mm(a, b):
    return a.to(F64) @ b.to(F64), a.to(F64).abs() @ b.to(F64).abs()


def test_projections_on_the_engine_operands(paper_run):
    """The encoder output and decoder input projections of one bf16 step at 8 images, on the operands the engine kept:
    logits = relu(enc) W + b (W as hi + lo, bias in the STORE product), z = y W_in + b (three products), dy = dz W_in^T,
    denc = dl W^T, the kernel and bias gradients onto non-zero bases, and the encoder output's ReLU backward."""
    s = paper_run["step"]
    n_hid, n_init, K = s["n_hid"], s["n_init"], K_PAPER
    rows = TRAIN_B * s["hw"] ** 2
    W = s["param/encoder/output/conv/kernel"].view(n_hid, K)
    b_e = s["param/encoder/output/conv/bias"]
    W_in = s["param/decoder/input/kernel"].view(K, n_init)
    b_d = s["param/decoder/input/bias"]
    hi = lambda t: t.to(BF16).float()
    a = s["enc_relu"].view(rows, n_hid)
    worst = 0.0
    # logits
    ref, absref = _mm(a, W)
    bound = dict(b=VK.SPLIT1 + (n_hid + 8) * UTC)
    name = f"logits = relu(enc) W + b rows={rows} {n_hid}->{K}"
    worst = max(worst, check(name, s["logits"], ref + b_e.to(F64), absref + b_e.abs().to(F64), **bound))
    must_fail(name + " bias twice", s["logits"], ref + 2 * b_e.to(F64), absref + b_e.abs().to(F64), **bound)
    r_hi, _ = _mm(a, hi(W))
    must_fail(name + " without lo", s["logits"], r_hi + b_e.to(F64), absref + b_e.abs().to(F64), **bound)
    del ref, absref, r_hi
    # z = y W_in + b
    y = s["y_out"]
    ref, absref = _mm(y, W_in)
    bound = dict(b=VK.SPLIT2 + (K + 8) * UTC)
    name = f"z = y W_in + b rows={rows} {K}->{n_init}"
    worst = max(worst, check(name, s["z_f32"], ref + b_d.to(F64), absref + b_d.abs().to(F64), **bound))
    must_fail(name + " bias twice", s["z_f32"], ref + 2 * b_d.to(F64), absref + b_d.abs().to(F64), **bound)
    r_hi, _ = _mm(hi(y), hi(W_in))
    must_fail(name + " without lo", s["z_f32"], r_hi + b_d.to(F64), absref + b_d.abs().to(F64), **bound)
    del ref, absref, r_hi
    # dy = dz W_in^T (dz exactly bf16, captured at the linear_wgrad that reads it)
    dz = s["dz"]
    ref, absref = _mm(dz, W_in.t())
    bound = dict(b=VK.SPLIT1 + (n_init + 8) * UTC)
    name = f"dy = dz W_in^T rows={rows} {n_init}->{K}"
    worst = max(worst, check(name, s["dy"], ref, absref, **bound))
    must_fail(name + " one row over", s["dy"], ref.roll(1, 0), absref.roll(1, 0), **bound)
    del ref, absref
    # denc = dl W^T
    dl = s["dlogits"]
    ref, absref = _mm(dl, W.t())
    bound = dict(b=VK.SPLIT2 + (K + 8) * UTC)
    name = f"denc = dl W^T rows={rows} {K}->{n_hid}"
    worst = max(worst, check(name, s["denc_f32"], ref, absref, **bound))
    must_fail(name + " one row over", s["denc_f32"], ref.roll(1, 0), absref.roll(1, 0), **bound)
    # the ReLU backward of the encoder output: the cast rounds denc to the nearest bf16 (within half an ulp, ties to
    # even) and the mask keeps it where enc_last > 0, so the result is bf16(denc) there and 0 elsewhere, bit for bit
    keep = s["enc_last"].view(rows, n_hid) > 0
    got = s["relu_bwd"].view(rows, n_hid)
    want = torch.where(keep, s["denc_f32"].to(BF16), torch.zeros((), dtype=BF16, device=DEV))
    assert torch.equal(got, want), "denc ReLU backward"
    assert not torch.equal(got, s["denc_f32"].to(BF16)), "denc ReLU backward: the mask drops nothing"
    print(f"[{TAG}] denc ReLU backward rows={rows} {n_hid}: bf16(denc) masked, bit-exact (worst err/bound 0)")
    del ref, absref, keep, want
    # gradients onto the seeded bases
    bases = s["bases"]
    for pname, x_op, g_op, L in (("encoder/output/conv", a, dl, rows), ("decoder/input", y, dz, rows)):
        base = bases[pname + "/kernel"]
        r, ra = _mm(x_op.t(), g_op)
        bound = dict(b=VK.SPLIT1 + (L + 64) * UTC)
        got = s[f"grad/{pname}/kernel"].view(base.shape)
        name = f"d {pname}/kernel rows={rows}"
        worst = max(worst, check(name, got, base.to(F64) + r, base.abs().to(F64) + ra, **bound))
        must_fail(name + " without its base", got, r, base.abs().to(F64) + ra, **bound)
        del r, ra
        bb = bases[pname + "/bias"]
        g64 = g_op.to(F64)
        name = f"d {pname}/bias rows={rows}"
        bound = dict(b=VK.SPLIT1 + 2 * (L + 64) * 2 * U + 8 * U)
        got = s[f"grad/{pname}/bias"]
        worst = max(worst, check(name, got, bb.to(F64) + g64.sum(0), bb.abs().to(F64) + g64.abs().sum(0), **bound))
        must_fail(name + " without its base", got, g64.sum(0), bb.abs().to(F64) + g64.abs().sum(0), **bound)
    print(f"[{TAG}] projections: worst err/bound {worst:.4f}")


# ------------------------------------------------------------------------------------------------------- real operands
def _conv_ref(kind, x, w, g, xshape, wshape):
    """float64 (ref, absref) of one convolution direction on the given operands (1 stride, SAME)."""
    out = []
    for xx, ww, gg in ((x, w, g), (None if x is None else x.abs(), None if w is None else w.abs(),
                                    None if g is None else g.abs())):
        if kind == "fwd":
            out.append(VK._conv64(xx.to(F64), ww.to(F64), 1, False))
        elif kind == "dgrad":
            xv = torch.zeros(xshape, dtype=F64, device=DEV, requires_grad=True)
            out.append(torch.autograd.grad(VK._conv64(xv, ww.to(F64), 1, False), xv, gg.to(F64))[0])
        else:
            wv = torch.zeros(wshape, dtype=F64, device=DEV, requires_grad=True)
            out.append(torch.autograd.grad(VK._conv64(xx.to(F64), wv, 1, False), wv, gg.to(F64))[0])
    return out


class RealOperands:
    """before / after hooks of a Recorder: clone each convolution's operands before it runs (the residual gradient
    before the launch overwrites it in place) and check its output against float64 of exactly those operands."""

    def __init__(self):
        self.worst = {}

    def before(self, entry, A):
        if entry not in CONV_ENTRIES:
            return None
        return {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in A.items()}

    def after(self, entry, A, S):
        if S is None:
            return
        c = S["c"]
        N, H, Cin, Cout, k = c.N, c.H, c.Cin, c.Cout, c.KH
        xshape, wshape = (N, H, H, Cin), (k, k, Cin, Cout)
        w = S.get("w", S.get("w_bf16"))
        if "fwd" in entry:
            ref, absref = _conv_ref("fwd", S["x"], w, None, xshape, wshape)
            ref, absref = ref + S["bias"].to(F64), absref + S["bias"].abs().to(F64)
            if c.relu:
                ref = ref.clamp_min(0)
            if S["residual"] is not None:
                ref, absref = ref + S["residual"].to(F64), absref + S["residual"].abs().to(F64)
            got, bound, muts = A["y"], dict(b=k * k * Cin * UTC + 8 * U, bf16_out=True), []
        elif "dgrad" in entry:
            ref, absref = _conv_ref("dgrad", None, w, S["dy"], xshape, wshape)
            keep = (S["x_mask"] > 0).to(F64) if S["x_mask"] is not None else 1.0
            add, add_abs = (S["dres"].to(F64), S["dres"].abs().to(F64)) if S["dres"] is not None else (0.0, 0.0)
            muts = []
            if S["x_mask"] is not None:
                muts.append(("mask dropped", ref + add, absref + add_abs))
            if S["dres"] is not None:
                muts.append(("dres dropped", ref * keep, absref * keep))
            ref, absref = ref * keep + add, absref * keep + add_abs
            got, bound = A["dx"], dict(b=k * k * Cout * UTC + 8 * U, bf16_out=True)
        else:
            ref, absref = _conv_ref("wgrad", S["x"], None, S["dy"], xshape, wshape)
            rel = ((A["dw"].to(F64) - S["dw"].to(F64) - ref).norm() / ref.norm().clamp_min(1e-300)).item()
            assert rel < VK.WGRAD_REL, (entry, xshape, wshape, rel)
            ref, absref = ref + S["dw"].to(F64), absref + S["dw"].abs().to(F64)
            got, bound, muts = A["dw"], dict(b=(N * H * H + 64) * UTC + 8 * U), []
        flags = "".join(f" {f}" for f in ("relu", "residual", "x_mask", "dres") if (f == "relu" and c.relu) or
                        (f != "relu" and S.get(f) is not None))
        if S.get("dres") is not None and _same(A["dres"], A["dx"]):
            flags += " in place"
        name = f"real B={N} {entry} {k}x{k} {Cin}->{Cout} @{H}{flags}"
        r = float64_bounds.worst_ratio(name, got, ref, absref, **bound)
        assert r < 1.0, f"{name}: worst err/bound {r:.4f}"
        for label, wref, wabs in muts:
            must_fail(f"{name} {label}", got, wref, wabs, **bound)
        self.worst[name] = max(self.worst.get(name, 0.0), r)


def test_real_operands_at_two_images(ops):
    """One bf16 step at the paper geometry with 2 images: every convolution launch against float64 of exactly what
    it read.  One line per launch class, with the worst ratio over its launches."""
    eng = paper_engine(seed=3, heavy_lo=False)
    img, u = step_inputs(eng, 2, 4)
    real = RealOperands()
    with Recorder(eng, before=real.before, after=real.after) as rec:
        train_step(eng, img, u)
        torch.cuda.synchronize()
    n = sum(l.entry in CONV_ENTRIES for l in rec.launches)
    assert n > 100 and len(real.worst) >= len(conv_classes(ops, rec.launches))
    for name, r in sorted(real.worst.items()):
        float64_bounds.report(name, r, TAG)
    print(f"[{TAG}] real operands B=2, {n} convolution launches: worst err/bound {max(real.worst.values()):.4f}")
