"""Launch census of every shipped DALL-E configuration: each kernel launch class that configs/dalle_*_b200.json makes
is replayed here against float64 or exempted to a named test that runs it at the recorded width or wider.

Recording.  Each configuration is built through dalle_model_fn (the path train_dalle.py runs, so every key is parsed
by the same helpers) at its per-GPU batch (the global batch over the data mesh axis, on mesh data:1), one layer per
distinct attention type of its schedule (products do not depend on the layer count), its recompute_grad, and a
random-init VAE stand-in of 1024 tokens.  One train_op, one eval_op, then DalleSampler on that engine: eager generate
and generate_graphed with top-k / top-p filtering at the per-GPU batch, and complete() with an image prefix, 2 samples
per prompt and guidance (prefill and hand-off).  Recording pauses inside the VAE's encode_tokens: the tokenizer's
launches are recorded at each configuration's real VAE and batch by test_vae_config_launches_gpu.py (the convolutional
network) and test_vae_paper_kernels_gpu.py (the DALL-E paper's network).  GEMMs are recorded at ops.gemm, everything
else at its outermost ops call.

Classes.  A GEMM class carries M, N, K, the operand majors, the mode, the output dtype, alpha != 1, every epilogue
input (bias, relu, residual, aux, colsum, dropout, ce_weights, gelu, z), split_k, n_valid < N, whether each of A, B
and D is read or written through a pitch wider than its extent, and each pointer's element offset in its storage mod
128.  Attention classes carry B, S, H, dh, scale, dropout and the radius / axial / conv geometry; the rest their
argument shapes, dtypes and flags.  Classes are deduplicated across configurations and replayed at the recorded shape,
so no shape mapping is needed.  Every replay runs under the same recorder and must launch each class it claims.
Each class also carries the phases it was launched in (train: train_op and eval_op; decode: the sampler's steps;
prefill: DalleEngine.prefill); the module ends with the worst err/bound of each family in each phase.

Bounds are those of the modules whose checkers run here (test_dalle_kernels_gpu.py, imported as DK, and the
GELU, weighted-loss, logits-mask, axial and convolutional attention modules).  The window products (GEMMs whose B or D
is a column window of a wider buffer: the logits mask's vocabulary dgrads and wgrads) read B from a full [d, Vpad]
buffer with NaN outside the window and accumulate D into a full fp32 buffer with a random base that must stay
bit-for-bit unchanged outside the window; two mutated references (the window shifted by 8 columns, the base dropped)
must fail the same bounds.

sqnorm / adam_step run at the parameter count one GPU updates at the configuration's own n_layers.  With
optimizer_state_sharding that is one data rank's ZeRO-1 shard, not every parameter: the 12B configuration's full
8.5e9 parameters do not fit one device four times in fp32 (test_zero1_gpu.py pins the sharded step to the replicated
one bit for bit).

Memory: comparisons run in DK.SLAB slabs, each case is freed before the next, and adam_step runs on slabs of the one
whole gradient, so that no test needs more of the shared device than test_dalle_kernels_gpu.py does.
"""
import collections
import gc
import glob
import math
import os
import time

import pytest
import torch

import float64_bounds
import launch_census as LC
import test_dalle_kernels_gpu as DK
from float64_bounds import DEV, U, UTC, nan_like

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
ROOT = DK.ROOT
TAG = "config-launches"
CONFIG_PATHS = sorted(glob.glob(os.path.join(ROOT, "configs", "dalle_*_b200.json")))
CONFIGS = [os.path.basename(p)[:-len(".json")] for p in CONFIG_PATHS]
VAE_SIZE = 64                    # the stand-in tokenizer: one stride-2 block, 64^2 -> 32 x 32 = 1024 tokens
PREFIX = 77                      # image codes of the complete() prompt (P = text_seq_len + 77, not a tile multiple)
WRAPPERS = ("linear_fwd", "linear_dgrad", "linear_wgrad")          # their gemm is recorded instead
HOST_ONLY = ("conv_desc", "conv_tc_supported", "conv_dgrad_tc_supported", "conv_wgrad_tc_supported", "ce_tiles",
             "attn_pairs", "attn_pairs_axial", "attn_pairs_conv")
_PEAK = [0]
_T0 = [0.0]


def report(name, r):
    return float64_bounds.report(name, r, TAG)


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    _T0[0] = time.time()
    yield _ops
    for ph in ("train", "decode", "prefill"):
        for (fam, p), r in sorted(_RATIOS.items()):
            if p == ph:
                print(f"[{TAG}] family {fam} ({ph}): worst err/bound {r:.4f}")
        rs = [r for (_, p), r in _RATIOS.items() if p == ph]
        if rs:
            print(f"[{TAG}] phase {ph}, every replayed family: worst err/bound {max(rs):.4f}")
    print(f"[{TAG}] module wall time {time.time() - _T0[0]:.0f} s, peak device memory {_PEAK[0] / 2 ** 30:.1f} GiB")


_TEST_PEAK = [0]


def case_peak():
    """Start a new peak-memory window for one case and return the peak of the window it closes (the test's own peak
    keeps the largest)."""
    peak = torch.cuda.max_memory_allocated()
    _TEST_PEAK[0] = max(_TEST_PEAK[0], peak)
    torch.cuda.reset_peak_memory_stats()
    return peak


@pytest.fixture(autouse=True)
def _peak_memory(request):
    """The comparisons run in DK.SLAB slabs and free each case before the next, so that no test needs more of the
    device than test_dalle_kernels_gpu.py does (shared machines)."""
    torch.cuda.reset_peak_memory_stats()
    _TEST_PEAK[0] = 0
    yield
    peak = max(torch.cuda.max_memory_allocated(), _TEST_PEAK[0])
    _PEAK[0] = max(_PEAK[0], peak)
    print(f"[{TAG}] {request.node.name}: peak device memory {peak / 2 ** 30:.1f} GiB")


# ------------------------------------------------------------------------------------------------------- classes
def _off(t):
    return None if t is None else t.storage_offset() % 128


def _sig(v):
    if isinstance(v, torch.Tensor):
        return (tuple(v.shape), str(v.dtype).replace("torch.", ""))
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    if isinstance(v, (tuple, list)):
        return tuple(_sig(x) for x in v)
    return type(v).__name__


def _kind(A):
    if A.get("conv") is not None:
        return "conv"
    if A.get("axial") is not None:
        return "axial"
    if A.get("radius") is not None:
        return "local"
    return "causal"


def _geo(v):
    return None if v is None else tuple(int(x) for x in v)


def describe(entry, A):
    """(class, info) of one ops call (None for the linear_* wrappers); info keeps what a replay needs beyond the class
    (pitches, storage offsets, n_valid, dropout descriptors), or is None."""
    from dalle_mtf_b200 import lib as L
    if entry in WRAPPERS:
        return None
    if entry == "gemm":
        a, b, out = A["a"], A["b"], A["out"]
        M, N, K = A["M"], A["N"], A["K"]
        lda = a.stride(0) if A["lda"] is None else A["lda"]
        ldb = b.stride(0) if A["ldb"] is None else A["ldb"]
        ldd = 0 if out is None else (out.stride(0) if A["ldd"] is None else A["ldd"])
        n_valid = int(A["n_valid"])
        cls = LC.launch_class(
            "gemm", M=M, N=N, K=K, a_mn=bool(A["a_mn"]), b_mn=bool(A["b_mn"]), mode=int(A["mode"]),
            out=None if out is None else str(out.dtype).replace("torch.", ""),
            alpha=float(A["alpha"]) != 1.0, bias=A["bias"] is not None, relu=bool(A["relu"]),
            residual=A["residual"] is not None, aux=A["aux"] is not None, colsum=A["colsum"] is not None,
            dropout=A["dropout"] is not None, ce_weights=A["ce_weights"] is not None, gelu=A["gelu"],
            z=A["z"] is not None, split_k=int(A["split_k"]), n_valid_lt_n=0 < n_valid < N,
            a_strided=lda > (M if A["a_mn"] else K), b_strided=ldb > (N if A["b_mn"] else K),
            d_strided=out is not None and ldd > N, a_off=_off(a), b_off=_off(b), d_off=_off(out))
        info = dict(lda=lda, ldb=ldb, ldd=ldd, n_valid=n_valid, alpha=float(A["alpha"]),
                    b_storage=b.storage_offset(), d_storage=None if out is None else out.storage_offset())
        if A["dropout"] is not None:
            info["dropout"] = A["dropout"]
        return cls, info
    if entry in ("attn_fwd", "attn_bwd"):
        cls = LC.launch_class(entry, kind=_kind(A), B=A["B"], S=A["S"], H=A["H"], dh=A["dh"], scale=float(A["scale"]),
                              dropout=A["dropout"] is not None, radius=A["radius"], axial=_geo(A["axial"]),
                              conv=_geo(A["conv"]))
        return cls, dict(dropout=A["dropout"])
    if entry in ("attn_decode", "attn_decode_dev"):
        rows, S, H, dh = A["qkv_step"].shape[0], *A["k_cache"].shape[1:]
        return LC.launch_class(entry, kind=_kind(A), rows=rows, S=S, H=H, dh=dh, scale=float(A["scale"]),
                               radius=A["radius"], axial=_geo(A["axial"]), conv=_geo(A["conv"])), None
    if entry in ("layernorm_fwd", "layernorm_bwd"):
        x = A["x"]
        f = dict(rows=x.shape[0], d=x.shape[1])
        if entry == "layernorm_bwd":
            f.update(dres=A["dres"] is not None, dxsum=A["dxsum"] is not None, dropout=A["dropout"] is not None)
        return LC.launch_class(entry, **f), dict(dropout=A.get("dropout"))
    if entry in ("embed_fwd", "embed_bwd"):
        ids = A["ids"]
        V = (A["wte"] if entry == "embed_fwd" else A["dwte"]).shape[0]
        f = dict(B=ids.shape[0], S=ids.shape[1], V=V, d=(A["wte"] if entry == "embed_fwd" else A["dwte"]).shape[1],
                 dropout=A["wte_drop"] is not None)
        return LC.launch_class(entry, **f), dict(wte_drop=A["wte_drop"], wpe_drop=A["wpe_drop"])
    if entry == "sqnorm":
        return LC.launch_class(entry, n=A["g"].numel()), None
    if entry == "adam_step":
        return LC.launch_class(entry, n=A["p"].numel(), clip=A["gnorm_sq"] is not None,
                               wd=float(A["weight_decay"]) != 0,
                               bias_correction=bool(A["bias_correction"]), zero_grad=bool(A["zero_grad"])), None
    return LC.launch_class(entry, **{k: _sig(v) for k, v in A.items() if k not in ("pos",)}), None


class Recorder(LC.OpsRecorder):
    def __init__(self):
        super().__init__(describe, nested=("gemm",), skip=HOST_ONLY)


# ------------------------------------------------------------------------------------------------------- recording
def _schedule(cfg):
    from dalle_mtf_b200.model_fns import attention_layers
    types, _ = attention_layers(cfg)
    return list(dict.fromkeys(types)) if types else ["global"]


def _params(cfg):
    from collections import defaultdict
    from dalle_mtf_b200.utils import parse_mesh
    mesh, _ = parse_mesh(cfg["mesh_shape"], cfg["layout"])
    B = cfg["train_batch_size"] // mesh.get("data", 1)
    types = _schedule(cfg)
    p = defaultdict(lambda: None, cfg)
    p.update(train_batch_size=B, eval_batch_size=B, mesh_shape="data:1", n_layers=len(types),
             attention_types=[[types, 1]] if cfg.get("attention_types") else None, model_path=None, iterations=1,
             vae_random_init=True, dataset={"image_size": VAE_SIZE},
             vae_params=defaultdict(lambda: None, {"model_type": "vae", "num_tokens": cfg["image_vocab_size"],
                                                   "convblocks": [[1, 32]], "dataset": {"image_size": VAE_SIZE}}))
    return p, B


def record_config(config):
    """(classes in first-launch order, {class: info}, per-GPU batch, n_params of the full configuration)."""
    from dalle_mtf_b200.input_fns import synthetic_captions
    from dalle_mtf_b200.model_fns import TRAIN, dalle_model_fn
    from dalle_mtf_b200.sampling import DalleSampler
    cfg = DK._config(config)
    p, B = _params(cfg)
    g = torch.Generator().manual_seed(B)
    feats = torch.rand(B, VAE_SIZE, VAE_SIZE, 3, generator=g) * 2 - 1
    caps = synthetic_captions(B, cfg["text_seq_len"], cfg["text_vocab_size"] - 1, g,
                              vocab=min(50257, cfg["text_vocab_size"]))
    with Recorder() as rec:
        rec.tag = "train"
        spec = dalle_model_fn(None, None, TRAIN, p)
        eng, vae = spec.engine, spec.extra["vae"]
        assert vae.image_seq_len == 1024 and eng.S == cfg["text_seq_len"] + 1024
        encode = vae.encode_tokens

        def paused_encode(*a, **k):
            rec.paused += 1
            try:
                return encode(*a, **k)
            finally:
                rec.paused -= 1
        vae.encode_tokens = paused_encode
        prefill = eng.prefill

        def tagged_prefill(*a, **k):
            rec.tag = "prefill"
            try:
                return prefill(*a, **k)
            finally:
                rec.tag = "decode"
        eng.prefill = tagged_prefill
        spec.train_op(feats, caps)
        spec.eval_op(feats, caps)
        torch.cuda.synchronize()
        rec.tag = "decode"
        smp = DalleSampler(eng, padding_id=cfg.get("padding_id"))
        text = caps.to(DEV, I32)
        torch.manual_seed(0)
        smp.generate(text, top_k=64, top_p=0.9)
        smp.generate_graphed(text, top_k=64, top_p=0.9)
        nb = max(1, B // 2)
        prefix = vae.encode_tokens(feats[:nb].to(DEV))[:, :PREFIX]
        smp.complete(text[:nb], image_prefix=prefix, samples_per_prompt=2, guidance_scale=3.0, top_k=64, top_p=0.9)
        torch.cuda.synchronize()
    # the wrappers above close over bound methods of eng and vae: a reference cycle that would keep this
    # configuration's engine on the device until the next garbage collection
    del eng.prefill, vae.encode_tokens
    n_full = _full_param_count(cfg, eng)
    classes, info = rec.classes(), dict(rec.info)
    for c, t in rec.tags.items():
        _TAGS.setdefault(c, set()).update(t)
    del smp, spec, eng, vae, rec
    gc.collect()
    torch.cuda.empty_cache()
    return classes, info, B, n_full


def _full_param_count(cfg, eng):
    """The flat parameter count of the configuration at its own n_layers (the recorded engine has one layer per
    distinct attention type; every layer has the same parameters)."""
    per_layer = sum(-(-math.prod(shape) // 64) * 64 for name, (_, shape) in eng.layout.entries.items()
                    if name.startswith("l0."))
    return eng.layout.size + (cfg["n_layers"] - eng.L) * per_layer


_CENSUS = {}
_TAGS = {}          # class -> phases it was launched in: "train" (train_op, eval_op), "decode", "prefill"
_RATIOS = {}        # (family, phase) -> worst err/bound of the replays of its classes


@pytest.fixture(scope="module")
def census(ops):
    """config -> (classes, info, B, n_full); recorded once per module."""
    if not _CENSUS:
        for c in CONFIGS:
            _CENSUS[c] = record_config(c)
    return _CENSUS


def note(family, classes, r):
    """Record the worst err/bound r of a replay that covered `classes` under each phase they were launched in."""
    for c in classes:
        for ph in _TAGS.get(c, ()):
            _RATIOS[(family, ph)] = max(_RATIOS.get((family, ph), 0.0), r)
    return r


def all_classes(census):
    """Distinct classes over every configuration, with the info of their first launch."""
    out = {}
    for c in CONFIGS:
        classes, info, _, _ = census[c]
        for k in classes:
            out.setdefault(k, info.get(k, {}))
    return out


# ------------------------------------------------------------------------------------------------------- routing
def _lib():
    from dalle_mtf_b200 import lib as L
    return L


def _gemm(c):
    return c[0] == "gemm"


def _plain_fields(f):
    return not (f["gelu"] or f["ce_weights"] or f["z"])


def is_plain_gemm(c):
    """Products DK.run_gemm_case replays: every field it ignores at its default, contiguous operands."""
    if not _gemm(c):
        return False
    f, L = LC.fields(c), _lib()
    return f["mode"] in (L.EPI_STORE, L.EPI_ATOMIC, L.EPI_RELU_BWD) and _plain_fields(f) and not f["alpha"] and \
        not (f["a_strided"] or f["b_strided"] or f["d_strided"])


def is_window_gemm(c):
    if not _gemm(c):
        return False
    f, L = LC.fields(c), _lib()
    return f["mode"] in (L.EPI_STORE, L.EPI_ATOMIC) and _plain_fields(f) and not f["alpha"] and not f["a_strided"] \
        and (f["b_strided"] or f["d_strided"]) and not (f["bias"] or f["residual"] or f["dropout"] or f["colsum"])


def is_cross_entropy(c):
    if c[0] in ("ce_finish", "ce_finish_weighted", "logits_mask_partition"):
        return True
    if not _gemm(c):
        return False
    f, L = LC.fields(c), _lib()
    return f["mode"] in (L.EPI_CE_STATS, L.EPI_CE_GRAD) and not f["gelu"] and not f["z"] and not f["a_strided"]


def is_gelu_gemm(c):
    return _gemm(c) and LC.fields(c)["gelu"] is not None and not LC.fields(c)["b_strided"]


def is_attention(c):
    return c[0] in ("attn_fwd", "attn_bwd")


CHECKERS = [
    ("test_plain_gemm_classes", is_plain_gemm),
    ("test_window_products", is_window_gemm),
    ("test_cross_entropy_classes", is_cross_entropy),
    ("test_gelu_classes", is_gelu_gemm),
    ("test_attention_classes", is_attention),
    ("test_layernorm_classes", lambda c: c[0] in ("layernorm_fwd", "layernorm_bwd")),
    ("test_embedding_classes", lambda c: c[0] in ("embed_fwd", "embed_bwd")),
    ("test_sqnorm_and_adam_at_the_full_parameter_count", lambda c: c[0] in ("sqnorm", "adam_step")),
]

# entry point (or entry:kind) -> (test id that pins it, why that covers the recorded class[, within]): within(fields)
# is true for the recorded shapes the named test covers; a class outside it is not exempted.  Every id is checked
# against pytest's collection by test_dalle_config_launches_cpu.py.
_DEC_WIDTHS = {(4, 128), (16, 64), (32, 128)}            # (H, dh) of test_decode_kernels_gpu.CONFIGS


def _rows(f, arg):
    return f[arg][0][0]


EXEMPT = {
    "cast_f32_to_bf16": ("test_abi_limits_gpu.py::test_flat_casts_and_split_past_2_31_elements",
                         "bf16 RNE of each element, bit for bit over 2^31 + 37 elements (the bf16 shadow refresh)",
                         lambda f: f["src"][0][0] <= 2 ** 31 + 37),
    "assemble_tokens": ("test_guidance_gpu.py::test_assemble_tokens_caption_drop_matches_the_oracle",
                        "integer concatenation, bit for bit; each element is one copy whatever the batch"),
    "assemble_tokens_pp": ("test_paper_embedding_gpu.py::test_assemble_tokens_pp_matches_the_oracle",
                           "integer concatenation with per-position pads, bit for bit; one copy per element"),
    "shift_labels": ("test_kernels_gpu.py::test_embedding_fwd_bwd_and_label_shift",
                     "integer shift, exact; also the label source of every cross-entropy replay here"),
    "logits_mask_scatter": ("test_logits_mask_gpu.py::test_partition_and_scatter_are_torch_indexing[1-256-1024-512]",
                            "row copies, bit for bit at S = 1280 and d = 512; rows are independent copies",
                            lambda f: f["dx"] is None or f["dx"][0][1] <= 512),
    "pos_compose": ("test_paper_embedding_gpu.py::test_pos_compose_is_the_bf16_rounded_definition[256-32-512]",
                    "bf16 RNE of one sum, bit for bit at TL 256, W 32, d 512",
                    lambda f: f["wpe"][0] == (256, 512) and f["image_row"][0] == (32, 512)),
    "pos_fold": ("test_paper_embedding_gpu.py::test_pos_fold_against_float64_and_reproducible[256-32-512]",
                 "per element against float64 at TL 256, W 32, d 512",
                 lambda f: f["dwpe"][0] == (256, 512) and f["dimage_row"][0] == (32, 512)),
    "kv_cache_fill": ("test_decode_kernels_gpu.py::test_hand_off_copies_at_production_widths",
                      "16-byte copies, bit for bit at H x dh up to 32 x 128 and P up to 1279",
                      lambda f: f["k_cache"][0][1] <= 1280 and f["k_cache"][0][2] * f["k_cache"][0][3] <= 4096),
    "rows_repeat": ("test_decode_kernels_gpu.py::test_hand_off_copies_at_production_widths",
                    "16-byte row copies, bit for bit"),
    "incr_i32": ("test_sampling_gpu.py::test_graph_replayed_generation_equals_eager_generation_when_greedy",
                 "the device position each replayed step advances: a wrong increment makes the replayed tokens differ "
                 "from eager generation"),
    "embed_fwd_at": ("test_decode_kernels_gpu.py::test_embedding_at_one_position",
                     "bf16 RNE of one sum, bit for bit at each configuration's width (one block per row)",
                     lambda f: f["wte"][0][1] in (512, 1024, 4096)),
    "embed_fwd_at_dev": ("test_decode_kernels_gpu.py::test_embedding_at_one_position",
                         "the device-position twin of embed_fwd_at, bit for bit",
                         lambda f: f["wte"][0][1] in (512, 1024, 4096)),
    "sample_rows_filtered": ("test_sampling_filter_gpu.py::test_kept_set_and_selection_match_the_float64_oracle",
                             "rows 1-130 at n 512 and 8192 (test_abi_limits_gpu.py at 51200)",
                             lambda f: _rows(f, "logits") <= 130 and f["hi"] - f["lo"] <= 8192),
    "sample_rows_filtered_at": ("test_sampling_filter_gpu.py::test_kept_set_and_selection_match_the_float64_oracle",
                                "the device-position twin, rows 1-130 at n 512 and 8192",
                                lambda f: _rows(f, "logits") <= 130 and f["hi"] - f["lo"] <= 8192),
    "sample_rows_guided": ("test_guidance_gpu.py::test_guided_draws_match_the_float32_oracle",
                           "1-130 guided rows (twice as many logits rows) at n 512 and 8192",
                           lambda f: _rows(f, "logits") <= 260 and f["hi"] - f["lo"] <= 8192),
    "attn_decode:causal": ("test_decode_kernels_gpu.py::test_attn_decode_sweep",
                           "rows 1, 64 and 130 at each configuration's H x dh, every cache position class",
                           lambda f: f["rows"] <= 130 and (f["H"], f["dh"]) in _DEC_WIDTHS and f["S"] == 1280),
    "attn_decode_dev:causal": ("test_decode_kernels_gpu.py::test_attn_decode_sweep",
                               "the device-position twin of attn_decode, at the same rows and widths",
                               lambda f: f["rows"] <= 130 and (f["H"], f["dh"]) in _DEC_WIDTHS and f["S"] == 1280),
    "attn_decode:local": ("test_local_kernels_gpu.py::test_attn_decode_local_sweep",
                          "rows up to 130 at each configuration's H x dh, radii up to 257",
                          lambda f: f["rows"] <= 130 and (f["H"], f["dh"]) in _DEC_WIDTHS and f["radius"] <= 257),
    "attn_decode_dev:local": ("test_local_kernels_gpu.py::test_attn_decode_local_sweep",
                              "the device-position twin, rows up to 130",
                              lambda f: f["rows"] <= 130 and (f["H"], f["dh"]) in _DEC_WIDTHS and f["radius"] <= 257),
    # the axial / conv decode tests run 4 rows: the kernel's grid is (H, rows), one block per (row, head) reading
    # only its own row's cache, so the row count adds blocks, not arithmetic; H x dh = 512 and the 256 + 32^2 grid
    # are the recorded ones
    "attn_decode:axial": ("test_axial_attention_gpu.py::test_attn_decode_axial_against_float64",
                          "both axes at H x dh = 512 on the 256 + 32^2 grid; one block per (row, head)",
                          lambda f: f["H"] * f["dh"] == 512 and f["axial"][:2] == (256, 32)),
    "attn_decode_dev:axial": ("test_axial_attention_gpu.py::test_attn_decode_axial_against_float64",
                              "the device-position twin, checked equal to attn_decode there",
                              lambda f: f["H"] * f["dh"] == 512 and f["axial"][:2] == (256, 32)),
    "attn_decode:conv": ("test_conv_attention_gpu.py::test_attn_decode_conv_against_float64",
                         "k 5, 11 and 40 at H x dh = 512 on the 256 + 32^2 grid; one block per (row, head)",
                         lambda f: f["H"] * f["dh"] == 512 and f["conv"][:2] == (256, 32)
                         and f["conv"][2] in (5, 11, 40)),
    "attn_decode_dev:conv": ("test_conv_attention_gpu.py::test_attn_decode_conv_against_float64",
                             "the device-position twin, checked equal to attn_decode there",
                             lambda f: f["H"] * f["dh"] == 512 and f["conv"][:2] == (256, 32)
                             and f["conv"][2] in (5, 11, 40)),
}


def make_census(present=None):
    return LC.Census(CHECKERS, EXEMPT, present if present is not None else set(globals()))


def routed(census, name):
    """{class: info} of the recorded classes the census hands to test `name`."""
    cen = make_census()
    return {c: i for c, i in all_classes(census).items() if cen.checker(c) == name}


def replayed(run):
    """Classes launched by run() (under the module's recorder)."""
    with Recorder() as rec:
        run()
        torch.cuda.synchronize()
    return set(rec.classes())


OFFSETS = ("a_off", "b_off", "d_off")


def _strip(c, ignore):
    return tuple(x for x in c if not (isinstance(x, tuple) and x[0] in ignore))


def claimed(want, got, ignore=()):
    """The classes of want that the replay launched (got)."""
    got = {_strip(c, ignore) for c in got}
    return [c for c in want if _strip(c, ignore) in got]


def assert_covered(name, want, got, ignore=()):
    """Every class in want was launched by the replay (got); ignore: fields not compared (the pointer alignments of
    replays whose operands are allocated by the checker they reuse)."""
    got = {_strip(c, ignore) for c in got}
    missing = [c for c in want if _strip(c, ignore) not in got]
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
        n_chk = sum(k in checked for k in classes)
        n_ex = sum(k in exempt for k in classes)
        print(f"[{TAG}] {c}: {len(classes)} classes recorded, {n_chk} checked here, {n_ex} exempted")
    print(f"[{TAG}] all configurations: {len(everything)} distinct classes, {len(checked)} checked here, "
          f"{len(exempt)} exempted")
    assert not unchecked, "recorded launch classes that nothing checks:\n" + "\n".join(map(str, unchecked))
    assert not stale, f"exemptions no recorded class answers to: {stale}"


# ------------------------------------------------------------------------------------------------------- GEMM
def _dk_desc(c):
    """The DK descriptor tuple of a plain class (see DK._describe)."""
    f = LC.fields(c)
    return ("gemm", f["M"], f["N"], f["K"], f["a_mn"], f["b_mn"], f["mode"],
            None if f["out"] is None else "torch." + f["out"], f["bias"], f["relu"], f["residual"], f["aux"],
            f["split_k"], 0, f["colsum"], f["dropout"])


def _place(t, off):
    """t copied into fresh storage at element offset `off` mod 128 (the recorded pointer alignment); the caller's
    reference to t is the only other one, so the original is freed when the caller rebinds it."""
    if t is None or off is None or off == 0:
        return t
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device=t.device)
    v = buf[off:].view(t.shape)
    v.copy_(t)
    return v


def replay_plain_gemm(ops, c, info, seed, tag=TAG):
    """One plain product class (is_plain_gemm) at its recorded shape through DK's operands and check_gemm, its
    operands at the recorded storage alignment.  Returns (worst err/bound, case name)."""
    f = LC.fields(c)
    desc = _dk_desc(c)
    splits = DK.gemm_splits(f["M"], f["N"], f["K"], f["mode"], f["split_k"], DK._sm())
    o = DK.gemm_operands(ops, desc, f["M"], f["K"], seed=seed, dropout=info.get("dropout"))
    o.a, o.b, o.out = _place(o.a, f["a_off"]), _place(o.b, f["b_off"]), _place(o.out, f["d_off"])
    DK.run_gemm(ops, o)
    tiles = -(-f["M"] // 128) * -(-f["N"] // 128) * splits
    name = DK.gemm_case_name(desc, f["M"], f["N"], f["K"], splits, tiles, info.get("dropout"))
    return DK.check_gemm(f"{tag} {name}", o, splits), name


def test_plain_gemm_classes(ops, census):
    """Every plain product (training, eval, decode, prefill) at its recorded shape through DK's operands and
    check_gemm, its operands at the recorded storage alignment."""
    want = routed(census, "test_plain_gemm_classes")
    assert want
    worst, peaks = 0.0, []

    def run():
        nonlocal worst
        for i, (c, info) in enumerate(want.items()):
            case_peak()
            held = torch.cuda.memory_allocated()
            r, name = replay_plain_gemm(ops, c, info, seed=i)
            worst = max(worst, note("GEMM", [c], r))
            torch.cuda.synchronize()
            peaks.append((torch.cuda.max_memory_allocated(), name, held))
    assert_covered("plain GEMM", want, replayed(run))
    peak, name, held = max(peaks)
    print(f"[{TAG}] family GEMM ({len(want)} classes): worst err/bound {worst:.4f}; largest case peak "
          f"{peak / 2 ** 30:.1f} GiB at {name} ({held / 2 ** 30:.1f} GiB held when it started)")


# ------------------------------------------------------------------------------------------------------- windows
def _windowed(rows, ld, c0, n, off, dtype, g, scale=1.0, outside=math.nan):
    """A full [rows, ld] buffer whose column window [c0, c0 + n) is random (scale) and whose other columns hold
    `outside`, placed so that the window's first element sits at storage offset `off` mod 128.  (parent, window)"""
    pad = (off - c0) % 128
    buf = torch.full((pad + rows * ld,), outside, dtype=dtype, device=DEV)
    parent = buf[pad:].view(rows, ld)
    parent[:, c0:c0 + n] = (torch.randn(rows, n, generator=g, device=DEV) * scale).to(dtype)
    return parent, parent[:, c0:c0 + n]


def window_products(ops, tag, T_text, T_image, K, io, V, Vpad, *, b_off=(0, 0), d_off=(0, 0), seed=0):
    """The four vocabulary products of the logits mask's backward in engine order (text block, then image block):
    dx = dlogits @ W[:, c0:c0+N]^T (B from a full NaN-outside wout) and G[:, c0:c0+N] += hf^T @ dlogits into one full
    fp32 buffer with a random base.  Checked per element with DK's bounds; outside the windows the buffer must be
    bit-for-bit the base; the overlap columns carry base + both blocks.  Returns (worst, worst of each mutant)."""
    L = _lib()
    c0i = io // 8 * 8
    blocks = [(T_text, 0, (io + 7) // 8 * 8), (T_image, c0i, (V - c0i + 7) // 8 * 8)]
    g = DK._gen(seed + T_image + io)
    base_buf, _ = _windowed(K, Vpad, 0, Vpad, d_off[0], F32, g)
    G = base_buf
    base = G.clone()
    sm = DK._sm()
    dw_ref = base.to(F64)
    dw_abs = torch.zeros(K, Vpad, dtype=F64, device=DEV)
    coef = torch.zeros(Vpad, dtype=F64, device=DEV)     # the largest b of the products that add onto each column
    worst, mut = 0.0, {"window +8": 0.0, "no base": 0.0}
    done = []
    for k, (rows, c0, N) in enumerate(blocks):
        if rows == 0:
            continue
        hf = DK._randn(rows, K, g=g, dtype=BF16)
        dl = DK._randn(rows, N, g=g, scale=2.0 ** -10, dtype=BF16)
        W, Wwin = _windowed(K, Vpad, c0, N, b_off[k], BF16, g, scale=0.02)
        dx = nan_like((rows, K), BF16)
        ops.linear_wgrad(hf, dl, G[:, c0:c0 + N])
        ops.linear_dgrad(dl, Wwin, dx)
        # dgrad: the STORE bound with K = the N window columns; the mutant reads the window 8 columns over
        name = f"{tag} dgrad {'text' if k == 0 else 'image'} {rows}x{K}x{N} c0={c0}"
        w = DK.Worst(name)
        lo = c0 + 8 if c0 + 8 + N <= Vpad else c0 - 8
        Wm = torch.nan_to_num(W[:, lo:lo + N].to(F64))
        W64 = Wwin.to(F64)
        for r0, r1 in DK._slabs(rows, max(N, K)):
            d64 = dl[r0:r1].to(F64)
            ref, absref = d64 @ W64.t(), d64.abs() @ W64.abs().t()
            w.add(dx[r0:r1], ref, absref, a=2 * U, b=(N + 9) * UTC, bf16_out=True)
            mut["window +8"] = max(mut["window +8"], float64_bounds.worst_ratio(
                name + " mutant", dx[r0:r1], d64 @ Wm.t(), absref, a=2 * U, b=(N + 9) * UTC, bf16_out=True))
        worst = max(worst, w.report())
        # wgrad: this block's contribution and its |.| graph, (rows + 8 + splits) UTC each
        splits = DK.gemm_splits(K, N, rows, L.EPI_ATOMIC, 0, sm)
        h64 = hf.to(F64)
        contrib = torch.zeros(K, N, dtype=F64, device=DEV)
        cabs = torch.zeros(K, N, dtype=F64, device=DEV)
        for r0, r1 in DK._slabs(rows, max(N, K)):
            contrib += h64[r0:r1].t() @ dl[r0:r1].to(F64)
            cabs += h64[r0:r1].abs().t() @ dl[r0:r1].to(F64).abs()
        b = (rows + 8 + splits) * UTC
        dw_ref[:, c0:c0 + N] += contrib
        dw_abs[:, c0:c0 + N] += b * cabs
        coef[c0:c0 + N] = coef[c0:c0 + N].clamp_min(b)
        done.append((c0, N, contrib))
        del hf, dl, W, Wwin, Wm, W64, dx, h64, cabs
    dw_abs += coef * base.abs().to(F64)
    cover = coef > 0
    assert torch.equal(G[:, ~cover].view(I32), base[:, ~cover].view(I32)), f"{tag}: wgrad wrote outside its windows"
    overlap = (done[0][0] + done[0][1] - done[-1][0]) if len(done) == 2 else 0
    nm = f"{tag} wgrad text then image into one [{K}, {Vpad}] buffer ({overlap} overlap columns)"
    r = float64_bounds.worst_ratio(nm, G[:, cover], dw_ref[:, cover], dw_abs[:, cover], a=2 * U, b=1.0)
    worst = max(worst, report(nm, r))
    shifted = base.to(F64)
    for c0, N, contrib in done:
        lo = c0 + 8 if c0 + 8 + N <= Vpad else c0 - 8
        shifted[:, lo:lo + N] += contrib
    mut["window +8"] = max(mut["window +8"], float64_bounds.worst_ratio(
        nm + " mutant", G[:, cover], shifted[:, cover], dw_abs[:, cover], a=2 * U, b=1.0))
    mut["no base"] = float64_bounds.worst_ratio(nm + " mutant", G[:, cover], (dw_ref - base.to(F64))[:, cover],
                                                dw_abs[:, cover], a=2 * U, b=1.0)
    return worst, mut


def _mask_shape(cfg):
    io = cfg["text_vocab_size"]
    V = io + cfg["image_vocab_size"] + 1
    return io, V, (V + 63) // 64 * 64


def test_window_products(ops, census):
    """The logits mask's four vocabulary products per element, at each masked configuration's recorded shape with the
    recorded pointer alignments, and at an image_offset = 7 (mod 8) shape; both mutants must fail."""
    want = routed(census, "test_window_products")
    masked = [c for c in CONFIGS if DK._config(c).get("logits_mask")]
    assert masked and want
    worst = 0.0
    got = set()
    for config in masked:
        cfg = DK._config(config)
        B = census[config][2]
        io, V, Vpad = _mask_shape(cfg)
        S, TL, K = cfg["text_seq_len"] + 1024, cfg["text_seq_len"], cfg["n_embd"]
        c0 = io // 8 * 8
        Nt = (io + 7) // 8 * 8
        rows = (B * (TL - 1), B * (S - TL + 1))
        # recorded alignments of W[:, c0:] (dgrad B) and G[:, c0:] (wgrad D), text block then image block
        b_off, d_off = [0, 0], [0, 0]
        for c in want:
            f = LC.fields(c)
            if f["b_strided"] and f["M"] in rows:
                b_off[0 if f["K"] == Nt else 1] = f["b_off"]
            if f["d_strided"] and f["K"] in rows:
                d_off[0 if f["N"] == Nt else 1] = f["d_off"]
        # one buffer: both wgrads' D windows lie in it, so the text window's alignment fixes the image one
        assert (d_off[0] + c0) % 128 == d_off[1], d_off
        res = {}

        def run():
            res["r"] = window_products(ops, f"{config} masked products B={B}", B * (TL - 1), B * (S - TL + 1), K, io,
                                       V, Vpad, b_off=b_off, d_off=d_off, seed=B)
        got |= replayed(run)
        r, mut = res["r"]
        worst = max(worst, note("window products", [c for c in want], r))
        for n, v in mut.items():
            print(f"[{TAG}] {config} masked products mutant {n}: worst err/bound {v:.3g} (must exceed 1)")
            assert v > 1.0, f"{config}: the window products also satisfy the mutant {n}"
    assert_covered("window products", want, got)
    # image_offset = 7 (mod 8): the image window starts 7 columns into an 8-column group
    # the window pointers where an engine would put them: W and G at offset 0, the image window c0 = 3000 columns in
    r, mut = window_products(ops, "masked products io=3007", 3 * 31, 3 * 65, 256, 3007, 3068, 3072,
                             b_off=(0, 3000 % 128), d_off=(0, 3000 % 128), seed=7)
    worst = max(worst, r)
    for n, v in mut.items():
        print(f"[{TAG}] io=3007 mutant {n}: worst err/bound {v:.3g} (must exceed 1)")
        assert v > 1.0
    print(f"[{TAG}] family window products: worst err/bound {worst:.4f}")


# ------------------------------------------------------------------------------------------------------- CE
def test_cross_entropy_classes(ops, census):
    """The vocabulary head of each configuration at its recorded T, K, V and Vpad through the checker of its flavour:
    DK.run_cross_entropy (CE_STATS -> ce_finish -> CE_GRAD), the weighted loss's run_weighted_ce, or the logits mask's
    run_windowed_ce (partition -> both blocks' CE_STATS / finish / CE_GRAD) at the recorded batch."""
    import test_logits_mask_gpu as LM
    import test_loss_weights_gpu as LW
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.model_fns import loss_weights
    want = routed(census, "test_cross_entropy_classes")
    got, worst, done = set(), collections.defaultdict(float), set()
    for config in CONFIGS:
        classes, info, B, _ = census[config]
        cfg = DK._config(config)
        S, TL = cfg["text_seq_len"] + 1024, cfg["text_seq_len"]
        stats = [c for c in classes if c in want and _gemm(c) and LC.fields(c)["mode"] == L.EPI_CE_STATS]
        weights, z = loss_weights(cfg)
        if cfg.get("logits_mask"):
            flavour, key = "masked", ("masked", B, cfg["n_embd"], cfg["text_vocab_size"], cfg["image_vocab_size"])
        else:
            (c,) = stats
            f = LC.fields(c)
            T, K, Vpad, V = f["M"], f["K"], f["N"], info[c]["n_valid"]
            flavour = "weighted" if weights is not None or z > 0 else "plain"   # (CE_STATS takes no weights)
            key = (flavour, T, K, V, Vpad, weights, z)
        if key in done:
            continue
        done.add(key)
        res = {}
        if flavour == "masked":
            run = lambda: LM.run_windowed_ce(ops, f"{TAG} {config} windowed CE B={B}", B, S, TL, cfg["n_embd"],
                                             cfg["text_vocab_size"], cfg["image_vocab_size"])
        else:
            g = DK._gen(T + K)
            h, W, bias, _, _ = DK.ce_operands(T, K, V, Vpad, g, dominate_cols=[0, V // 2, V - 2, V - 1])
            tokens = DK.synthetic_tokens(cfg, T // S, g)
            labels = torch.empty_like(tokens)
            ops.shift_labels(tokens, labels, V - 1)
            labels = labels.view(T).contiguous()
            if flavour == "weighted":
                run = lambda: LW.run_weighted_ce(ops, f"{TAG} {config} weighted CE T={T}", T, K, V, Vpad, S, TL,
                                                 labels=labels, h=h, W=W, bias=bias, weights=weights, z=z,
                                                 global_batch=B)
            else:
                run = lambda: DK.run_cross_entropy(ops, f"{TAG} {config} CE T={T} V={V}", T, K, V, Vpad,
                                                   labels=labels, h=h, W=W, bias=bias)
        got_now = replayed(lambda: res.setdefault("r", run()))
        got |= got_now
        worst[flavour] = max(worst[flavour], note("cross-entropy " + flavour, claimed(want, got_now, OFFSETS),
                                                   res["r"]))
    # the replays allocate their own operands: pointer alignments are not compared
    assert_covered("cross-entropy", want, got, OFFSETS)
    for n, r in worst.items():
        print(f"[{TAG}] family cross-entropy ({n}): worst err/bound {r:.4f}")


# ------------------------------------------------------------------------------------------------------- GELU
def test_gelu_classes(ops, census):
    import test_gelu_gpu as GE
    want = routed(census, "test_gelu_classes")
    got, worst, done = set(), 0.0, set()
    for c in want:
        f = LC.fields(c)
        M = f["M"]
        d, N = f["K"], f["N"]                            # fwd [M, d] x [d, 4d]; bwd [M, d] x [4d, d]^T
        if (M, d, N) in done:
            continue
        done.add((M, d, N))
        res = {}
        got_now = replayed(lambda: res.setdefault("r", GE._epilogue_case(ops, f"{TAG} gelu M={M}", M, d, N,
                                                                         seed=M + d)))
        got |= got_now
        worst = max(worst, note("GELU", claimed(want, got_now, OFFSETS), res["r"]))
    assert_covered("GELU", want, got, OFFSETS)
    print(f"[{TAG}] family GELU ({len(done)} shapes): worst err/bound {worst:.4f}")


# ------------------------------------------------------------------------------------------------------- attention
def test_attention_classes(ops, census):
    """Causal (with and without dropout), local, axial and convolutional attention at the recorded B, S, H, dh."""
    import test_axial_attention_gpu as AX
    import test_conv_attention_gpu as CV
    import test_local_attention_gpu as LA
    import test_local_kernels_gpu as LK
    want = routed(census, "test_attention_classes")
    got, worst, done = set(), 0.0, set()
    for c, info in want.items():
        f = LC.fields(c)
        key = (f["kind"], f["B"], f["S"], f["H"], f["dh"], f["scale"], f["dropout"], f["axial"], f["conv"])
        if key in done:
            continue
        done.add(key)
        B, S, H, dh, scale = f["B"], f["S"], f["H"], f["dh"], f["scale"]
        qkv, dout = DK._qkv(B, S, H, dh, DK._gen(B * S + H))
        tag = f"{TAG} {f['kind']} attention B={B} S={S} H={H} dh={dh}" + (" dropout" if f["dropout"] else "")
        res = {}
        if f["kind"] == "causal":
            drop = info.get("dropout")
            got_now = replayed(lambda: res.setdefault("r", DK.run_attention(ops, tag, B, S, H, dh, scale, qkv, dout,
                                                                            dropout=drop)))
            got |= got_now
            worst = max(worst, note("attention", claimed(want, got_now), res["r"]))
            continue
        if f["kind"] == "local":
            r = f["radius"]
            got_now = replayed(lambda: res.setdefault("o", LA.run_local(ops, qkv, dout, r, scale)))
            got |= got_now
            out, lse, dqkv = res["o"]
            worst = max(worst, note("attention", claimed(want, got_now), LK.check_local(
                f"{tag} r={r}", qkv, out, lse, r, dout, dqkv, scale=scale)))
            continue
        mod, geo = (AX, f["axial"]) if f["kind"] == "axial" else (CV, f["conv"])
        runner = AX.run_axial if f["kind"] == "axial" else CV.run_conv
        got_now = replayed(lambda: res.setdefault("o", runner(ops, qkv, dout, geo, scale)))
        got |= got_now
        out, lse, dqkv = res["o"]
        mask = mod.visible(S, *geo)
        rs = collections.defaultdict(float)
        for b0 in range(0, B, 2):
            for n, v in mod.ratios(qkv[b0:b0 + 2], dout[b0:b0 + 2], out[b0:b0 + 2], lse[b0:b0 + 2], dqkv[b0:b0 + 2],
                                   mask, scale).items():
                rs[n] = max(rs[n], v)
        worst = max(worst, note("attention", claimed(want, got_now), max(report(f"{tag} {n}", v)
                                                                         for n, v in rs.items())))
    assert_covered("attention", want, got)
    print(f"[{TAG}] family attention: worst err/bound {worst:.4f}")


# ------------------------------------------------------------------------------------------------------- LayerNorm
def test_layernorm_classes(ops, census):
    want = routed(census, "test_layernorm_classes")
    got, worst, done = set(), 0.0, set()
    for c, info in want.items():
        f = LC.fields(c)
        if c[0] == "layernorm_fwd":
            key = (f["rows"], f["d"], True, True, None)
        else:
            key = (f["rows"], f["d"], f["dres"], f["dxsum"], info.get("dropout") is not None)
        if key in done:
            continue
        done.add(key)
        rows, d, dres, dxsum, _ = key
        drop = info.get("dropout")
        res = {}
        got_now = replayed(lambda: res.setdefault("r", DK.run_layernorm(
            ops, f"{TAG} LN rows={rows} d={d} dres={int(dres)} dxsum={int(dxsum)}" + (" dropout" if drop else ""),
            rows, d, dres=dres, dxsum=dxsum, dropout=drop, seed=rows + d)))
        got |= got_now
        worst = max(worst, note("LayerNorm", claimed(want, got_now), res["r"]))
    assert_covered("LayerNorm", want, got)
    print(f"[{TAG}] family LayerNorm: worst err/bound {worst:.4f}")


# ------------------------------------------------------------------------------------------------------- embedding
def test_embedding_classes(ops, census):
    want = routed(census, "test_embedding_classes")
    got, worst, done = set(), 0.0, set()
    for c, info in want.items():
        f = LC.fields(c)
        key = (f["B"], f["S"], f["V"], f["d"], f["dropout"])
        if key in done:
            continue
        done.add(key)
        B, S, V, d, _ = key
        g = DK._gen(V + B * S)
        ids = torch.randint(0, V, (B, S), generator=g, device=DEV, dtype=I32)
        ids[:, 40:256] = V // 2                          # long runs of one (padding) id, as the captions have
        res = {}
        got_now = replayed(lambda: res.setdefault("r", DK.run_embedding(
            ops, f"{TAG} embedding B={B} S={S} V={V} d={d}" + (" dropout" if f["dropout"] else ""), ids, V, d, 1.0, g,
            wte_drop=info.get("wte_drop"), wpe_drop=info.get("wpe_drop"))))
        got |= got_now
        worst = max(worst, note("embedding", claimed(want, got_now), res["r"]))
    assert_covered("embedding", want, got)
    print(f"[{TAG}] family embedding: worst err/bound {worst:.4f}")


# ------------------------------------------------------------------------------------------------------- Adam
def test_sqnorm_and_adam_at_the_full_parameter_count(ops, census):
    """sqnorm / adam_step with the flags each configuration passes, at the parameter count one GPU updates with the
    configuration's own n_layers (the recorded engine has fewer layers, and the partial-sum depth of sqnorm's bound
    grows with n).  That is every parameter, except with optimizer_state_sharding: there one data rank's ZeRO-1 shard,
    since the 12B configuration's full count (8.5e9) does not fit one device in fp32 four times over."""
    from dalle_mtf_b200.utils import parse_mesh
    want = routed(census, "test_sqnorm_and_adam_at_the_full_parameter_count")
    flags = {}
    for config in CONFIGS:
        classes, _, _, n_full = census[config]
        cfg = DK._config(config)
        n = n_full
        if cfg.get("optimizer_state_sharding"):
            data = parse_mesh(cfg["mesh_shape"], cfg["layout"])[0].get("data", 1)
            n = -(-n_full // data)
        for c in classes:
            if c in want and c[0] == "adam_step":
                f = LC.fields(c)
                flags.setdefault((n, f["clip"], f["wd"], f["bias_correction"], f["zero_grad"]), (config, []))
                flags[(n, f["clip"], f["wd"], f["bias_correction"], f["zero_grad"])][1].append(c)
    assert flags
    worst = 0.0
    for (n, clip, wd, bc, zg), (config, cls) in flags.items():
        sq = [c for c in want if c[0] == "sqnorm"]
        worst = max(worst, note("Adam", cls + sq, _adam_case(ops, f"{config} n={n}", n, clip, wd, bc, zg)))
    print(f"[{TAG}] family Adam ({len(flags)} flag sets): worst err/bound {worst:.4f}")


ADAM_SLAB = 1 << 25


def _adam_inputs(i0, i1, seed):
    """p, m, v, g of elements [i0, i1), drawn from a generator of their own slab (regenerated for the check)."""
    g = DK._gen(seed * 1000003 + i0 // ADAM_SLAB)
    k = i1 - i0
    sign = lambda: torch.where(torch.rand(k, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    logu = lambda lo, hi: torch.exp(torch.empty(k, device=DEV).uniform_(math.log(lo), math.log(hi), generator=g))
    p = torch.randn(k, generator=g, device=DEV) * 0.05
    gr = sign() * logu(1e-8, 1e-3)
    m = sign() * logu(1e-9, 1e-4)
    v = logu(1e-18, 1e-8)
    return p, m, v, gr


def _adam_case(ops, tag, n, clip, wd, bc, zg):
    """sqnorm over the whole n-element gradient, then adam_step on ADAM_SLAB-element slabs of it with that norm, each
    slab checked (DK.check_adam_update) and freed before the next: only the gradient is ever held whole.  adam_step
    is elementwise, so a slab's elements see the arithmetic of one n-element launch (test_abi_limits_gpu.py runs one
    launch past 2^31 elements)."""
    slabs = [(i, min(n, i + ADAM_SLAB)) for i in range(0, n, ADAM_SLAB)]
    seed = n % 9973
    gd = torch.empty(n, device=DEV)
    for i0, i1 in slabs:
        gd[i0:i1] = _adam_inputs(i0, i1, seed)[3]
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-6
    wdv, clipv = (0.01 if wd else 0.0), (0.05 if clip else 0.0)
    gn_base = 1e-3
    gn = torch.full((1,), gn_base, device=DEV)
    ops.sqnorm(gd, gn)
    sq = gn_base + sum((gd[i0:i1].to(F64) ** 2).sum() for i0, i1 in slabs)
    worst = [DK.check(f"{TAG} sqnorm {tag}", gn, sq.reshape(1), sq.reshape(1), a=0.0, b=DK.sqnorm_depth(n) * U)]
    step = 3 if bc else 0
    for i0, i1 in slabs:
        p, m, v, gr = _adam_inputs(i0, i1, seed)
        pd, md, vd = p.clone(), m.clone(), v.clone()
        p16 = nan_like((i1 - i0,), BF16)
        ops.adam_step(pd, md, vd, gd[i0:i1], p16, lr, b1, b2, eps, wdv, gn if clip else None, clipv, 1.0, bc, step,
                      zero_grad=zg)
        DK.check_adam_update(f"{tag} [{i0}, {i1})", (p, m, v, gr, gn), (pd, md, vd, p16), lr, b1, b2, eps, wdv, clipv,
                             1.0, bc, step, worst=worst)
        assert (gd[i0:i1] == 0).all() if zg else torch.equal(gd[i0:i1], gr)
        del p, m, v, gr, pd, md, vd, p16
    return max(worst)
