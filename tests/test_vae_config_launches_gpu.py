"""Launch census of every shipped convolutional dVAE configuration: each kernel launch class that a
configs/vae_*_b200.json with the convolutional network (VaeEngine) makes is replayed here against float64 at the
recorded shape, or exempted to a named test that runs it at the recorded K and flags on at least as many rows.

Recording.  Each configuration is built through vae_model_fn at its per-GPU batch (the global batch over the data mesh
axis, on mesh data:1), with every other key of the configuration (K, convblocks, Gumbel hardness, KL, logit-Laplace,
recompute).  Phases, each a tag of the classes launched in it:
  train     two train_ops (the first step of a KL anneal has weight 0); the launches between dp.begin_overlap() and
            dp.wait() are tagged backward
  eval      one eval_op of an EVAL-mode model (eval Gumbel is hard where train Gumbel is soft)
  tokenize  encode_tokens at the per-GPU train batch of every DALL-E b200 configuration whose vae_model names this VAE
  decode    decode_tokens at those configurations' predict_batch_size, which generate_dalle.py decodes in one call
            (the engine runs it in passes of at most decode_pass_images() images)
The batches are read from the configurations (phase_batches).  GEMMs are recorded at ops.gemm with the DALL-E census's
fields (test_dalle_config_launches_gpu.py, imported as CL); convolutions carry their descriptor, the kernel (tc or
direct) and the forward flags (relu, bias, residual), the dgrad flags (mask, dres, in place) or the wgrad's dbias;
every other entry its argument shapes and flags (CL.describe).

Replays run under the same recorder and must launch each class they claim.  Bounds are those of
test_vae_kernels_gpu.py (VK), test_dalle_kernels_gpu.py (DK) and the modules named in EXEMPT.  Each convolution is
replayed through VK.run_conv at the recorded N with exactly the recorded variants (float64 references in image slabs);
the backward classes of configurations with a data axis > 1 run again with DataParallel.MAX_CTAS SMs reserved, the
reservation the overlapped all-reduce makes, which changes the wgmma grids and the wgrad pixel splits.  One bf16 train
step per geometry at 2 images checks every convolution and GEMM launch against float64 of exactly the operands it
read.  Every check runs a mutated reference that must fail.

The module ends with the worst err/bound of each family in each phase, its wall time and its peak device memory.
"""
import gc
import glob
import json
import math
import os
import time

import pytest
import torch

import float64_bounds
import launch_census as LC
import test_dalle_config_launches_gpu as CL
import test_dalle_kernels_gpu as DK
import test_vae_kernels_gpu as VK
from float64_bounds import DEV, U, UTC, nan_like

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
ROOT = DK.ROOT
TAG = "vae-config-launches"
CONV_ENTRIES = ("conv2d_fwd", "conv2d_fwd_tc", "conv2d_dgrad", "conv2d_dgrad_tc", "conv2d_wgrad", "conv2d_wgrad_tc")
BIT_EXACT = ("cast_f32_to_bf16", "cast_bf16_to_f32", "split_f32", "onehot_rows", "argmax_rows")
PHASES = ("train", "backward", "eval", "tokenize", "decode")
_PEAK = [0]
_T0 = [0.0]


def _load(path):
    with open(path) as f:
        return json.load(f)


def _name(path):
    return os.path.basename(path)[:-len(".json")]


def _config(name):
    return _load(os.path.join(ROOT, "configs", name + ".json"))


def is_conv_network(cfg):
    from dalle_mtf_b200.model_fns import vae_architecture
    return vae_architecture(cfg, cfg["dataset"]["image_size"]) is None


CONFIGS = [_name(p) for p in sorted(glob.glob(os.path.join(ROOT, "configs", "vae_*_b200.json")))
           if is_conv_network(_load(p))]
DALLE_CONFIGS = [_name(p) for p in sorted(glob.glob(os.path.join(ROOT, "configs", "dalle_*_b200.json")))]


def data_axis(cfg):
    from dalle_mtf_b200.utils import parse_mesh
    return parse_mesh(cfg["mesh_shape"], cfg["layout"])[0].get("data", 1)


def phase_batches(vae):
    """phase -> the batches one call of that phase runs with: the per-GPU train and eval batches of the VAE
    configuration, the per-GPU train batch (tokenize) and the predict_batch_size (decode, one decode_tokens call) of
    every DALL-E b200 configuration whose vae_model is `vae`."""
    cfg = _config(vae)
    users = [_config(d) for d in DALLE_CONFIGS if _config(d)["vae_model"] == vae]
    return {"train": [cfg["train_batch_size"] // data_axis(cfg)], "eval": [cfg["eval_batch_size"] // data_axis(cfg)],
            "tokenize": sorted({c["train_batch_size"] // data_axis(c) for c in users}),
            "decode": sorted({c["predict_batch_size"] for c in users})}


def report(name, r):
    return float64_bounds.report(name, r, TAG)


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    _T0[0] = time.time()
    yield _ops
    for ph in PHASES + ("backward, SMs reserved",):
        for (fam, p), r in sorted(_RATIOS.items()):
            if p == ph:
                print(f"[{TAG}] family {fam} ({ph}): worst err/bound {r:.4f}")
    print(f"[{TAG}] module wall time {time.time() - _T0[0]:.0f} s, peak device memory {_PEAK[0] / 2 ** 30:.1f} GiB")


@pytest.fixture(autouse=True)
def _peak_memory(request):
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated()
    _PEAK[0] = max(_PEAK[0], peak)
    print(f"[{TAG}] {request.node.name}: peak device memory {peak / 2 ** 30:.1f} GiB")


# ------------------------------------------------------------------------------------------------------- classes
def conv_fields(entry, A):
    """The class fields of one convolution launch: descriptor, kernel and the flags of its role."""
    c = A["c"]
    f = dict(N=c.N, H=c.H, W=c.W, Cin=c.Cin, Cout=c.Cout, k=c.KH, stride=c.stride, transposed=bool(c.transposed),
             f32=bool(c.act_f32), kernel="tc" if entry.endswith("_tc") else "direct")
    if "fwd" in entry:
        f.update(relu=bool(c.relu), bias=A["bias"] is not None, residual=A["residual"] is not None)
    elif "dgrad" in entry:
        f.update(mask=A["x_mask"] is not None, dres=A["dres"] is not None,
                 in_place=A["dres"] is not None and A["dres"].data_ptr() == A["dx"].data_ptr())
    else:
        f.update(dbias=A.get("dbias") is not None)
    return f


def describe(entry, A):
    if entry in CONV_ENTRIES:
        return LC.launch_class(entry, **conv_fields(entry, A)), None
    if entry == "conv2d_first_fwd":
        N, H, W, _ = A["x_f32"].shape
        return LC.launch_class(entry, N=N, H=H, W=W, Cout=A["y_bf16"].shape[-1]), None
    return CL.describe(entry, A)


class Recorder(LC.OpsRecorder):
    def __init__(self, before=None, after=None):
        super().__init__(describe, nested=("gemm",), skip=CL.HOST_ONLY, before=before, after=after)


# ------------------------------------------------------------------------------------------------------- recording
def _params(cfg, mode):
    from collections import defaultdict
    B = cfg[f"{mode}_batch_size"] // data_axis(cfg)
    p = defaultdict(lambda: None, cfg)
    p.update(train_batch_size=B, eval_batch_size=B, mesh_shape="data:1", model_path=None)
    return p, B


def record_config(vae):
    """(classes in first-launch order, {class: info}) of one configuration's four phases."""
    from dalle_mtf_b200.model_fns import EVAL, TRAIN, vae_model_fn
    cfg = _config(vae)
    batches = phase_batches(vae)
    size = cfg["dataset"]["image_size"]
    g = torch.Generator().manual_seed(len(vae))
    with Recorder() as rec:
        rec.tag = "train"
        p, B = _params(cfg, "train")
        spec = vae_model_fn(None, None, TRAIN, p)
        dp = spec.dp
        begin, wait = dp.begin_overlap, dp.wait

        def tagged_begin():
            rec.tag = "backward"
            return begin()

        def tagged_wait():
            out = wait()
            rec.tag = "train"
            return out
        dp.begin_overlap, dp.wait = tagged_begin, tagged_wait
        # two steps: under kl_anneal_steps the first step's KL weight is 0, which runs the plain Gumbel backward
        for _ in range(2):
            spec.train_op(torch.rand(B, size, size, 3, generator=g) * 2 - 1)
        torch.cuda.synchronize()
        del dp.begin_overlap, dp.wait, spec
        gc.collect()
        torch.cuda.empty_cache()
        rec.tag = "eval"
        p, B = _params(cfg, "eval")
        spec = vae_model_fn(None, None, EVAL, p)
        spec.eval_op(torch.rand(B, size, size, 3, generator=g) * 2 - 1)
        eng = spec.engine
        rec.tag = "tokenize"
        for Bt in batches["tokenize"]:
            eng.encode_tokens((torch.rand(Bt, size, size, 3, generator=g) * 2 - 1).to(DEV))
        rec.tag = "decode"
        for Bd in batches["decode"]:
            eng.decode_tokens(torch.randint(0, eng.K, (Bd, eng.image_seq_len), generator=g, dtype=I32).to(DEV))
        torch.cuda.synchronize()
    classes, info = rec.classes(), dict(rec.info)
    for c, t in rec.tags.items():
        _TAGS.setdefault(c, set()).update(t)
    del spec, eng, rec
    gc.collect()
    torch.cuda.empty_cache()
    return classes, info


_CENSUS = {}
_TAGS = {}          # class -> phases it was launched in
_RATIOS = {}        # (family, phase) -> worst err/bound of the replays of its classes


@pytest.fixture(scope="module")
def census(ops):
    if not _CENSUS:
        for c in CONFIGS:
            _CENSUS[c] = record_config(c)
    return _CENSUS


def note(family, classes, r, phase=None):
    """Record the worst err/bound r of a replay that covered `classes` under each phase they were launched in (or
    under `phase`)."""
    for c in classes:
        for ph in ([phase] if phase else _TAGS.get(c, ())):
            _RATIOS[(family, ph)] = max(_RATIOS.get((family, ph), 0.0), r)
    return r


def all_classes(census):
    out = {}
    for c in CONFIGS:
        classes, info = census[c]
        for k in classes:
            out.setdefault(k, info.get(k) or {})
    return out


# ------------------------------------------------------------------------------------------------------- routing
def is_plain_gemm(c):
    return CL.is_plain_gemm(c)


CHECKERS = [
    ("test_convolution_classes", lambda c: c[0] in CONV_ENTRIES or c[0] == "colsum"),
    ("test_first_layer_classes", lambda c: c[0] == "conv2d_first_fwd"),
    ("test_gemm_classes", is_plain_gemm),
    ("test_bit_exact_classes", lambda c: c[0] in BIT_EXACT),
    ("test_gumbel_classes", lambda c: c[0] in ("gumbel_softmax_fwd", "gumbel_softmax_bwd")),
    ("test_adam_classes", lambda c: c[0] == "adam_step"),
]


# entry point -> (test id, why it covers the recorded class, within(fields)): within is true for the recorded shapes
# the named test covers (the same K and flags on at least as many rows).  test_vae_config_launches_cpu.py checks that
# each id is collected and that each predicate rejects what its test does not run.
EXEMPT = {
    "vae_kl_stats": ("test_vae_kl_gpu.py::test_kl_stats_against_float64",
                     "per element against float64 at 16384 x 8192 and 32768 x 512; rows are independent blocks",
                     lambda f: (f["K"] == 8192 and f["rows"] <= 16384) or (f["K"] == 512 and f["rows"] <= 32768)),
    "gumbel_softmax_bwd_kl": ("test_vae_kl_gpu.py::test_kl_backward_against_float64",
                              "per element against float64 at 16384 x 8192 and 32768 x 512",
                              lambda f: (f["K"] == 8192 and f["rows"] <= 16384) or
                              (f["K"] == 512 and f["rows"] <= 32768)),
    "mse_fwd_bwd": ("test_vae_kernels_gpu.py::test_mse_loss_and_gradient",
                    "the gradient bit for bit and the loss sum against float64 over 32 x 256^2 x 3 elements",
                    lambda f: math.prod(f["pred"][0]) <= 32 * 256 * 256 * 3),
    "logit_laplace": ("test_vae_logit_laplace_gpu.py::test_logit_laplace_kernel_against_float64",
                      "training mode per element against float64 at 16 and 32 x 256^2 pixels of 3 channels",
                      lambda f: f["target"] is not None and f["Cp"] == 3 and f["n_pix"] <= 32 * 256 * 256),
}


def make_census(present=None):
    return LC.Census(CHECKERS, EXEMPT, present if present is not None else set(globals()))


def routed(census, name):
    cen = make_census()
    return {c: i for c, i in all_classes(census).items() if cen.checker(c) == name}


def replayed(run):
    with Recorder() as rec:
        run()
        torch.cuda.synchronize()
    return set(rec.classes())


def assert_covered(name, want, got):
    missing = [c for c in want if c not in got]
    assert not missing, f"{name}: recorded classes the replay did not launch: {missing}"


# ------------------------------------------------------------------------------------------------------- the census
def test_every_recorded_launch_is_checked(census):
    """A recorded class is replayed by a test of this module or exempted to a named test; an exemption no class
    answers to is stale."""
    cen = make_census()
    everything = all_classes(census)
    checked, exempt, unchecked, stale = cen.classify(everything)
    for c in CONFIGS:
        classes = census[c][0]
        print(f"[{TAG}] {c}: {len(classes)} classes recorded, {sum(k in checked for k in classes)} replayed here, "
              f"{sum(k in exempt for k in classes)} exempted; batches {phase_batches(c)}")
    print(f"[{TAG}] all configurations: {len(everything)} distinct classes, {len(checked)} replayed here, "
          f"{len(exempt)} exempted")
    assert not unchecked, "recorded launch classes that nothing checks:\n" + "\n".join(map(str, unchecked))
    assert not stale, f"exemptions no recorded class answers to: {stale}"


def test_direct_kernels_run_at_the_production_batch(census):
    """The direct-kernel classes (the training path's first conv, the decoder's 1x1 output conv and its dgrad, the
    direct wgrads) are recorded, and replayed here, at every configuration's per-GPU train batch."""
    everything = all_classes(census)
    for vae in CONFIGS:
        B = phase_batches(vae)["train"][0]
        direct = {c[0] for c in census[vae][0] if c[0] in CONV_ENTRIES and LC.fields(c)["kernel"] == "direct"
                  and LC.fields(c)["N"] == B}
        assert {"conv2d_fwd", "conv2d_dgrad", "conv2d_wgrad"} <= direct, (vae, B, direct)
    cen = make_census()
    assert all(cen.checker(c) == "test_convolution_classes" for c in everything if c[0] in CONV_ENTRIES)


# ------------------------------------------------------------------------------------------------------- convolutions
def conv_geometries(classes):
    """(N, H, Cin, Cout, k, stride, transposed, f32) -> recorded forward / dgrad variants (VK names) and wgrad."""
    out = {}
    for c in classes:
        if c[0] not in CONV_ENTRIES:
            continue
        f = LC.fields(c)
        assert f["H"] == f["W"], c
        d = out.setdefault((f["N"], f["H"], f["Cin"], f["Cout"], f["k"], f["stride"], f["transposed"], f["f32"]),
                           {"fwd": set(), "dgrad": set(), "wgrad": False})
        if "fwd" in c[0]:
            assert f["bias"] and not (f["relu"] and f["residual"]), c
            d["fwd"].add("relu" if f["relu"] else "res" if f["residual"] else "plain")
        elif "dgrad" in c[0]:
            parts = (["mask"] if f["mask"] else []) + ([("dres in place" if f["in_place"] else "dres")]
                                                       if f["dres"] else [])
            d["dgrad"].add(" ".join(parts) or "plain")
        else:
            d["wgrad"] = True
    return out


def replay_convolutions(ops, classes, label, seed=0, fwd=True):
    """VK.run_conv on every geometry of `classes` at its recorded N with exactly its recorded variants (fwd=False: the
    backward variants only).  Returns the worst err/bound."""
    worst = 0.0
    order = lambda s, names: tuple(v for v in names if v in s)
    for i, ((N, H, Cin, Cout, k, stride, tr, f32), d) in enumerate(sorted(conv_geometries(classes).items())):
        tag = f"{label} {k}x{k}{' T' if tr else ''} s{stride} {Cin}->{Cout} @{H} N={N}"
        worst = max([worst] + VK.run_conv(ops, tag, N, H, Cin, Cout, k, stride, tr, dgrad=bool(d["dgrad"]),
                                          wgrad=d["wgrad"], act_f32=f32, seed=seed + i,
                                          fwd_variants=order(d["fwd"], VK.FWD_VARIANTS) if fwd else (),
                                          dgrad_variants=order(d["dgrad"], VK.DGRAD_VARIANTS), line_tag=TAG))
        gc.collect()
        torch.cuda.empty_cache()
    return worst


def test_convolution_classes(ops, census):
    """Every convolution class (and the colsum of each wgmma wgrad's bias gradient) at its recorded N; the backward
    classes of configurations with a data axis > 1 again with DataParallel.MAX_CTAS SMs reserved."""
    from dalle_mtf_b200.dist import DataParallel
    want = routed(census, "test_convolution_classes")
    res = {}
    got = replayed(lambda: res.setdefault("r", replay_convolutions(ops, want, "conv")))
    assert_covered("convolutions", want, got)
    for c in want:
        note("convolution", [c], res["r"])
    print(f"[{TAG}] family convolution ({len(conv_geometries(want))} geometries): worst err/bound {res['r']:.4f}")
    bwd = {c for vae in CONFIGS if data_axis(_config(vae)) > 1 for c in census[vae][0]
           if c in want and "backward" in _TAGS.get(c, ()) and c[0] != "colsum"}
    if not bwd:
        return
    k = DataParallel.MAX_CTAS
    with float64_bounds.reserved_sms(k) as sm:
        got = replayed(lambda: res.update(r=replay_convolutions(ops, bwd, "conv", seed=500, fwd=False)))
    assert_covered("convolutions with SMs reserved", bwd, got)
    note("convolution", bwd, res["r"], phase="backward, SMs reserved")
    print(f"[reserved-sms k={k} sm={sm}] [{TAG}] family convolution, backward ({len(bwd)} classes): "
          f"worst err/bound {res['r']:.4f}")


def first_layer_case(ops, N, H, W, Cout, seed):
    """conv2d_first_fwd as test_vae_kernels_gpu.test_first_layer_convolution checks it (the image as bf16 hi + lo, the
    weights as bf16), compared a slab of images at a time; the reference without the lo half must fail."""
    from oracle import vae as OV
    g = VK._gen(seed)
    x = torch.rand(N, H, W, 3, generator=g, device=DEV) * 2 - 1
    w = VK._randn(4, 4, 3, Cout, g=g, scale=0.2)
    bias = VK._randn(Cout, g=g, scale=0.1)
    y = nan_like((N, H // 2, W // 2, Cout), BF16)
    ops.conv2d_first_fwd(x, w, bias, y)
    w64, b64 = w.to(BF16).to(F64), bias.to(F64)
    bound = dict(b=97 * UTC + 4 * U, bf16_out=True)
    name = f"first layer wgmma N={N} {H}x{W} Cout={Cout}"
    r = mut = 0.0
    per = max(1, VK.SLAB // (H * W * Cout // 4))
    for n0 in range(0, N, per):
        s = slice(n0, min(N, n0 + per))
        hi = x[s].to(BF16).float()
        lo = (x[s] - hi).to(BF16).float()
        ref = OV.conv2d_same(hi.to(F64) + lo.to(F64), w64, b64, 2)
        absref = OV.conv2d_same(hi.abs().to(F64) + lo.abs().to(F64), w64.abs(), bias.abs().to(F64), 2)
        r = max(r, float64_bounds.worst_ratio(name, y[s], ref, absref, **bound))
        mut = max(mut, float64_bounds.worst_ratio(name + " without lo", y[s], OV.conv2d_same(hi.to(F64), w64, b64, 2),
                                                  absref, **bound))
    assert mut >= 1.0, f"{name}: the reference without the image's lo half passes too ({mut:.4f})"
    return report(name, r)


def test_first_layer_classes(ops, census):
    """The tokenizer's first conv (fp32 image, fused cast) at each recorded N and Cout."""
    want = routed(census, "test_first_layer_classes")
    assert want
    res = {}

    def run():
        for i, c in enumerate(want):
            f = LC.fields(c)
            res[c] = first_layer_case(ops, f["N"], f["H"], f["W"], f["Cout"], seed=10 + i)
    assert_covered("first layer", want, replayed(run))
    for c, r in res.items():
        note("first layer", [c], r)


# ------------------------------------------------------------------------------------------------------- GEMM
def test_gemm_classes(ops, census):
    """The codebook products (bf16 hi / lo operands, fp32 out) at their recorded shapes through the DALL-E census's
    GEMM checker."""
    want = routed(census, "test_gemm_classes")
    assert want
    worst = 0.0

    def run():
        nonlocal worst
        for i, (c, info) in enumerate(want.items()):
            r, _ = CL.replay_plain_gemm(ops, c, info, seed=i, tag=TAG)
            worst = max(worst, note("GEMM", [c], r))
            gc.collect()
    assert_covered("GEMM", want, replayed(run))
    print(f"[{TAG}] family GEMM ({len(want)} classes): worst err/bound {worst:.4f}")


# ------------------------------------------------------------------------------------------------------- bit exact
def test_bit_exact_classes(ops, census):
    """The casts (round to nearest even), the hi + lo split, decode_tokens' one-hot rows with their offset and
    encode_tokens' first-maximum argmax, bit for bit at the recorded sizes."""
    want = routed(census, "test_bit_exact_classes")
    g = VK._gen(77)

    def run():
        for c in want:
            f = LC.fields(c)
            if c[0] in ("cast_f32_to_bf16", "split_f32"):
                shape = f["src"][0]
                x = torch.randn(shape, generator=g, device=DEV) * torch.exp2(
                    torch.randint(-12, 12, shape, generator=g, device=DEV).float())
                hi = nan_like(f["dst" if c[0] == "cast_f32_to_bf16" else "hi"][0], BF16)
                x = x.view(hi.shape)
                if c[0] == "split_f32":
                    lo = nan_like(f["lo"][0], BF16)
                    ops.split_f32(x, hi, lo)
                    assert torch.equal(lo.view(torch.int16), (x - x.to(BF16).float()).to(BF16).view(torch.int16)), c
                else:
                    ops.cast_f32_to_bf16(x, hi)
                assert torch.equal(hi.view(torch.int16), x.to(BF16).view(torch.int16)), c
            elif c[0] == "cast_bf16_to_f32":
                x = torch.randn(f["src"][0], generator=g, device=DEV).to(BF16)
                y = nan_like(f["dst"][0], F32)
                ops.cast_bf16_to_f32(x, y)
                assert torch.equal(y, x.float().view(y.shape)), c
            elif c[0] == "onehot_rows":
                (rows,), (_, K), off = f["idx"][0], f["y"][0], f["offset"]
                idx = (torch.randint(0, K, (rows,), generator=g, device=DEV) + off).to(I32)
                idx[:2] = torch.tensor([off, off + K - 1], device=DEV)         # both ends of the window
                y = nan_like((rows, K), F32)
                ops.onehot_rows(idx, y, off)
                want_y = torch.nn.functional.one_hot(idx.long() - off, K).float()
                assert torch.equal(y, want_y), c
                if off == 0:        # mutation: ids read one code over
                    assert not torch.equal(y, torch.nn.functional.one_hot((idx.long() + 1) % K, K).float())
            else:   # argmax_rows
                rows, K = f["rows"], f["K"]
                x = torch.randint(-3, 4, (rows, K), generator=g, device=DEV).float()      # many ties
                idx = torch.full((rows,), -1, dtype=I32, device=DEV)
                ops.argmax_rows(x, idx, rows, K)
                assert torch.equal(idx.long(), VK.first_argmax(x)), c
                last = K - 1 - VK.first_argmax(x.flip(-1))                    # mutation: the last maximum
                assert not torch.equal(idx.long(), last), c
            print(f"[{TAG}] {c[0]} {dict((k, v) for k, v in f.items() if v is not None)}: bit-exact "
                  f"(worst err/bound 0)")
    assert_covered("bit-exact", want, replayed(run))
    for c in want:
        note("bit-exact", [c], 0.0)


# ------------------------------------------------------------------------------------------------------- Gumbel
def test_gumbel_classes(ops, census):
    """Gumbel-softmax forward (soft and hard, with the recorded noise and temperature) and its straight-through
    backward at the recorded rows x K, with VK's references, compared in row slabs.  The forward's mutant drops the
    noise, the backward's the sum(y dy) term."""
    want = routed(census, "test_gumbel_classes")
    res = {}

    def run():
        for i, c in enumerate(want):
            f = LC.fields(c)
            rows, K, tau = f["rows"], f["K"], f["tau"]
            g = VK._gen(rows + K + i)
            logits = torch.randn(rows, K, generator=g, device=DEV) * 2
            per = max(1, DK.SLAB // K)
            if c[0] == "gumbel_softmax_fwd":
                u = VK._uniform_noise(rows, K, g) if f["u"] is not None else None
                y_soft, y_out = nan_like((rows, K), F32), nan_like((rows, K), F32)
                idx = torch.full((rows,), -1, dtype=I32, device=DEV)
                ops.gumbel_softmax_fwd(logits, u, y_soft, y_out, idx, rows, K, tau, f["hard"])
                name = f"gumbel fwd rows={rows} K={K} tau={tau:g} noise={int(u is not None)} hard={int(f['hard'])}"
                r = mut = 0.0
                for r0 in range(0, rows, per):
                    s = slice(r0, min(rows, r0 + per))
                    ref, bound = VK.gumbel_ref(logits[s], None if u is None else u[s], tau)
                    r = max(r, float64_bounds.worst_ratio(name, y_soft[s], ref, bound, a=0.0, b=1.0))
                    if u is not None:
                        ref0, _ = VK.gumbel_ref(logits[s], None, tau)
                        mut = max(mut, float64_bounds.worst_ratio(name, y_soft[s], ref0, bound, a=0.0, b=1.0))
                    assert torch.equal(idx[s].long(), VK.first_argmax(y_soft[s])), name
                    del ref, bound
                if u is not None:
                    assert mut >= 1.0, f"{name}: the reference without noise passes too ({mut:.4f})"
                if f["hard"]:
                    assert torch.equal(y_out, torch.nn.functional.one_hot(idx.long(), K).float()), name
                else:
                    assert torch.equal(y_out, y_soft), name
            else:
                y = nan_like((rows, K), F32)
                ops.gumbel_softmax_fwd(logits, None, y, None, None, rows, K, tau, False)
                dy = torch.randn(rows, K, generator=g, device=DEV)
                dl = nan_like((rows, K), F32)
                ops.gumbel_softmax_bwd(y, dy, dl, rows, K, tau)
                name = f"gumbel bwd rows={rows} K={K} tau={tau:g}"
                bound = dict(a=4 * U, b=(K / 32 + 8) * U, floor=2.0 ** -149 / tau)
                r = mut = 0.0
                for r0 in range(0, rows, per):
                    s = slice(r0, min(rows, r0 + per))
                    y64, d64 = y[s].to(F64), dy[s].to(F64)
                    dot = (y64 * d64).sum(-1, keepdim=True)
                    absref = y64 * (d64.abs() + (y64 * d64).abs().sum(-1, keepdim=True)) / tau
                    r = max(r, float64_bounds.worst_ratio(name, dl[s], y64 * (d64 - dot) / tau, absref, **bound))
                    mut = max(mut, float64_bounds.worst_ratio(name, dl[s], y64 * d64 / tau, absref, **bound))
                assert mut >= 1.0, f"{name}: the reference without sum(y dy) passes too ({mut:.4f})"
            res[c] = report(name, r)
    assert_covered("Gumbel", want, replayed(run))
    for c, r in res.items():
        note("Gumbel", [c], r)


# ------------------------------------------------------------------------------------------------------- Adam
def test_adam_classes(ops, census):
    """adam_step at each configuration's n_params_padded with the bf16 shadow, its lr and grad_scale = 1 / data (the
    cross-replica mean), at the first step (bias-corrected), through DK.check_adam_update."""
    want = routed(census, "test_adam_classes")
    worst, got = [], set()
    for vae in CONFIGS:
        cfg = _config(vae)
        mine = [c for c in census[vae][0] if c in want]
        if not mine:
            continue
        (c,) = mine
        f = LC.fields(c)
        n = f["n"]
        p, m, v, gr = CL._adam_inputs(0, n, n % 9973)
        pd, md, vd, gd = p.clone(), m.clone(), v.clone(), gr.clone()
        p16 = nan_like((n,), BF16)
        gscale = 1.0 / data_axis(cfg)
        lr = cfg["lr"]

        def run():
            ops.adam_step(pd, md, vd, gd, p16, lr, 0.9, 0.999, 1e-8, 0.0, None, 0.0, gscale, True, 1,
                          zero_grad=f["zero_grad"])
        got |= replayed(run)
        DK.check_adam_update(f"{TAG} {vae} n={n} grad_scale={gscale:g}", (p, m, v, gr, None), (pd, md, vd, p16), lr,
                             0.9, 0.999, 1e-8, 0.0, 0.0, gscale, True, 1, worst=worst)
        assert (gd == 0).all() if f["zero_grad"] else torch.equal(gd, gr)
        note("Adam", [c], worst[-1])
        del p, m, v, gr, pd, md, vd, gd, p16
    assert_covered("Adam", want, got)
    print(f"[{TAG}] family Adam: worst err/bound {max(worst):.4f}")


# ------------------------------------------------------------------------------------------------------- real operands
def _conv_ref(kind, S, c, w):
    """float64 (ref, absref) of one convolution direction of descriptor c on the operands S it read."""
    N, H, Cin, Cout, k, stride, tr = c.N, c.H, c.Cin, c.Cout, c.KH, c.stride, bool(c.transposed)
    wshape = (k, k, Cout, Cin) if tr else (k, k, Cin, Cout)
    out = []
    for sign in (lambda t: t, lambda t: t.abs()):
        if kind == "fwd":
            out.append(VK._conv64(sign(S["x"].to(F64)), sign(w.to(F64)), stride, tr))
        elif kind == "dgrad":
            xv = torch.zeros((N, H, H, Cin), dtype=F64, device=DEV, requires_grad=True)
            out.append(torch.autograd.grad(VK._conv64(xv, sign(w.to(F64)), stride, tr), xv, sign(S["dy"].to(F64)))[0])
        else:
            wv = torch.zeros(wshape, dtype=F64, device=DEV, requires_grad=True)
            out.append(torch.autograd.grad(VK._conv64(sign(S["x"].to(F64)), wv, stride, tr), wv,
                                           sign(S["dy"].to(F64)))[0])
    return out


class RealOperands:
    """before / after hooks of a Recorder: clone each convolution's and GEMM's operands before it runs (the residual
    gradient before the launch overwrites it in place, an accumulated output before the launch adds onto it) and check
    its output against float64 of exactly those operands, with a mutated reference that must fail."""

    def __init__(self):
        self.worst = {}
        self.launches = 0

    def before(self, entry, A):
        if entry not in CONV_ENTRIES and entry != "gemm":
            return None
        return {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in A.items()}

    def after(self, entry, A, S):
        if S is None:
            return
        self.launches += 1
        if entry == "gemm":
            return self._gemm(A, S)
        c = S["c"]
        f = conv_fields(entry, A)
        k = c.KH
        w = S.get("w", S.get("w_bf16"))
        taps = 4 if c.transposed else k * k
        if "fwd" in entry:
            ref, absref = _conv_ref("fwd", S, c, w)
            ref, absref = ref + S["bias"].to(F64), absref + S["bias"].abs().to(F64)
            if c.relu:
                ref = ref.clamp_min(0)
            if S["residual"] is not None:
                ref, absref = ref + S["residual"].to(F64), absref + S["residual"].abs().to(F64)
            got = A["y"]
            bound = dict(b=taps * c.Cin * UTC + 8 * U, bf16_out=got.dtype == BF16)
            muts = [("one pixel over", ref.roll(1, 2), absref.roll(1, 2))]
        elif "dgrad" in entry:
            ref, absref = _conv_ref("dgrad", S, c, w)
            keep = (S["x_mask"] > 0).to(F64) if S["x_mask"] is not None else 1.0
            add, add_abs = (S["dres"].to(F64), S["dres"].abs().to(F64)) if S["dres"] is not None else (0.0, 0.0)
            muts = []
            if S["x_mask"] is not None:
                muts.append(("mask dropped", ref + add, absref + add_abs))
            if S["dres"] is not None:
                muts.append(("dres dropped", ref * keep, absref * keep))
            ref, absref = ref * keep + add, absref * keep + add_abs
            if not muts:
                muts.append(("one pixel over", ref.roll(1, 2), absref.roll(1, 2)))
            got = A["dx"]
            bound = dict(b=k * k * c.Cout * UTC + 8 * U, bf16_out=got.dtype == BF16)
        else:
            ref, absref = _conv_ref("wgrad", S, c, None)
            rel = ((A["dw"].to(F64) - S["dw"].to(F64) - ref).norm() / ref.norm().clamp_min(1e-300)).item()
            assert rel < VK.WGRAD_REL, (entry, f, rel)
            ref, absref = ref + S["dw"].to(F64), absref + S["dw"].abs().to(F64)
            got = A["dw"]
            L_w = c.N * (c.H * c.H if c.transposed else (-(-c.H // c.stride)) ** 2)
            bound = dict(b=(L_w + 64) * UTC + 8 * U)
            muts = [("one output channel over", ref.roll(1, -1), absref.roll(1, -1))]
        flags = "".join(f" {n}" for n in ("relu", "residual", "mask", "dres", "in_place", "dbias") if f.get(n))
        name = (f"real B={c.N} {entry} {k}x{k}{' T' if c.transposed else ''} s{c.stride} {c.Cin}->{c.Cout} "
                f"@{c.H}{flags}")
        self._check(name, got, ref, absref, bound, muts)

    def _gemm(self, A, S):
        from dalle_mtf_b200 import lib as L
        M, N, K, mode = S["M"], S["N"], S["K"], S["mode"]
        assert mode in (L.EPI_STORE, L.EPI_ATOMIC) and S["bias"] is None and S["residual"] is None, (M, N, K, mode)
        a = S["a"].reshape(K, M).t() if S["a_mn"] else S["a"].reshape(M, K)
        b = S["b"].reshape(K, N) if S["b_mn"] else S["b"].reshape(N, K).t()
        a64, b64 = a.to(F64), b.to(F64)
        ref, absref = a64 @ b64, a64.abs() @ b64.abs()
        splits = DK.gemm_splits(M, N, K, mode, S["split_k"], DK._sm())
        if mode == L.EPI_ATOMIC:
            base = S["out"].reshape(M, N).to(F64)
            ref, absref = ref + base, absref + base.abs()
        bound = dict(a=2 * U, b=(K + 8 + splits) * UTC)
        name = f"real gemm {'ATOMIC' if mode == L.EPI_ATOMIC else 'STORE'} {M}x{N}x{K} aT={int(S['a_mn'])} " \
               f"bT={int(S['b_mn'])} splits={splits}"
        self._check(name, A["out"].reshape(M, N), ref, absref, bound,
                    [("one row over", ref.roll(1, 0), absref.roll(1, 0))])

    def _check(self, name, got, ref, absref, bound, muts):
        r = float64_bounds.worst_ratio(name, got, ref, absref, **bound)
        assert r < 1.0, f"{name}: worst err/bound {r:.4f}"
        for label, wref, wabs in muts:
            VK.must_fail(f"{name} {label}", got, wref, wabs, **bound)
        self.worst[name] = max(self.worst.get(name, 0.0), r)


def _geometries():
    """One configuration per distinct network: image size, convblocks, K, loss and KL (the step's launches depend on
    nothing else)."""
    seen = {}
    for vae in CONFIGS:
        cfg = _config(vae)
        key = (cfg["dataset"]["image_size"], json.dumps(cfg["convblocks"]), cfg["num_tokens"],
               cfg.get("reconstruction_loss"), cfg.get("kl_loss_weight") is not None)
        seen.setdefault(key, vae)
    return list(seen.values())


@pytest.mark.parametrize("vae", _geometries())
def test_real_operands_at_two_images(ops, vae):
    """One bf16 train step of the configuration's network (its image size, convblocks, K, loss and KL) at 2 images:
    every convolution and codebook-product launch against float64 of exactly what it read.  One line per launch
    class, with the worst ratio over its launches."""
    from dalle_mtf_b200.model_fns import build_vae_engine, vae_kl_weight, vae_temperature
    cfg = _config(vae)
    size = cfg["dataset"]["image_size"]
    eng = build_vae_engine(cfg, size, torch.device(DEV), kl=cfg.get("kl_loss_weight") is not None)
    eng.init_params(seed=3)
    g = VK._gen(4)
    img = torch.rand(2, size, size, 3, generator=g, device=DEV) * 2 - 1
    u = torch.rand(2 * eng.image_seq_len, eng.K, generator=g, device=DEV).clamp_(1e-9, 1 - 2.0 ** -24)
    real = RealOperands()
    hard = cfg.get("train_gumbel_hard")
    kl = vae_kl_weight(cfg.get("kl_anneal_steps") or 1, cfg)
    with Recorder(before=real.before, after=real.after):
        eng.zero_grads()
        eng.forward(img, u, vae_temperature(0, cfg), True if hard is None else hard, kl_weight=kl)
        eng.backward()
        torch.cuda.synchronize()
    assert real.launches > 40 and any("gemm" in n for n in real.worst) and any("wgrad" in n for n in real.worst)
    for name, r in sorted(real.worst.items()):
        report(name, r)
    print(f"[{TAG}] {vae} real operands B=2, {real.launches} launches: worst err/bound {max(real.worst.values()):.4f}")
    del eng


# ------------------------------------------------------------------------------------------------------- decoding
def test_decoding_in_passes_equals_one_pass(ops, monkeypatch):
    """decode_tokens of vae_coco_b200 at 12 images in one pass and in passes of 5, 5 and 2: every decode launch
    computes an image from its own codes alone (no split depends on the batch), so the two are equal bit for bit."""
    from dalle_mtf_b200 import vae_engine as VE
    from dalle_mtf_b200.model_fns import build_vae_engine
    cfg = _config("vae_coco_b200")
    eng = build_vae_engine(cfg, cfg["dataset"]["image_size"], torch.device(DEV))
    eng.init_params(seed=5)
    B = 12
    assert eng.decode_pass_images() >= B
    g = torch.Generator().manual_seed(6)
    idx = (torch.randint(0, eng.K, (B, eng.image_seq_len), generator=g, dtype=I32) + 9).to(DEV)
    one = eng.decode_tokens(idx, offset=9).clone()
    monkeypatch.setattr(VE, "DECODE_PASS_BYTES", 5 * eng.buffer_bytes(1))
    assert eng.decode_pass_images() == 5
    chunked = eng.decode_tokens(idx, offset=9)
    assert chunked.shape == one.shape and torch.equal(chunked, one)
    assert not torch.equal(chunked[5:], one[:-5])               # the passes land in their own images
    print(f"[{TAG}] decode_tokens B={B}: passes of 5, 5 and 2 equal one pass bit for bit (worst err/bound 0)")
