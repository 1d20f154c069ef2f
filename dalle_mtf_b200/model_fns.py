"""Step assembly — the drop-in boundary.  Mirrors src/model_fns.py (dalle_model_fn) and src/model_fns_tf.py
(vae_model_fn): same signature ``model_fn(features, labels, mode, params)``, same parameter keys, PREDICT raises
NotImplementedError (src/model_fns.py:135-136, src/model_fns_tf.py:29-30).

Where the reference returns a TPUEstimatorSpec wiring TF ops, these return a ``StepSpec``: the model_fn is called
ONCE (like the Estimator's graph build) and ``spec.train_op(features, labels)`` runs one optimisation step on a
batch (host or device tensors), returning the device scalar with the global-mean loss.  One process per GPU: each
rank passes ITS shard of the global batch (rows rank*B/N..., the reference's "batch_dim:data" layout).
"""
import math
import numbers

import torch

from . import lib as L
from . import ops
from .dalle_engine import ATTENTION_TYPES, DalleEngine, validate_activation, validate_conv_kernel, \
    validate_logits_mask, validate_loss_weights, validate_per_position_padding, validate_position_embedding, \
    validate_layer_scale, validate_rotary, validate_rotary_emb, validate_sandwich_norm, \
    validate_share_input_output_emb, validate_shared_ids, validate_shift_tokens, validate_stable, validate_block_sparse
from .dist import DataParallel
from .optimizers import OptimizerConfig
from .utils import latest_checkpoint, load_checkpoint, local_path, parse_mesh, print_n_params
from .vae_engine import RECONSTRUCTION_LOSSES, VaeEngine, codebook_usage
from .vae_paper_engine import PaperVaeEngine, check_paper_geometry
from .vqgan_engine import VqganEngine, check_vqgan_geometry

TRAIN, EVAL, PREDICT = "train", "eval", "predict"   # tf.estimator.ModeKeys values


def mode_to_str(mode):
    """src/utils/utils.py:29-37."""
    if mode in (TRAIN, EVAL, PREDICT):
        return mode
    raise ValueError(f"Invalid mode {mode}")


class StepSpec:
    """What model_fn hands back to the training loop (stands in for TPUEstimatorSpec)."""

    def __init__(self, mode, engine, train_op=None, eval_op=None, state_fn=None, load_fn=None, dp=None, extra=None):
        self.mode = mode
        self.engine = engine
        self.train_op = train_op      # (features, labels) -> device scalar loss (global mean)
        self.eval_op = eval_op        # (features, labels) -> device scalar loss
        self.state_fn = state_fn      # () -> checkpoint dict
        self.load_fn = load_fn        # (dict) -> None
        self.dp = dp
        self.global_step = 0
        self.extra = extra or {}
        self.loss = None              # device scalar of the last step (read it only when logging: it syncs)
        self.loss_parts = None        # weighted loss: device [3] = text-row mean CE, image-row mean CE, mean z-term;
                                      # VAE with KL: device [2] = reconstruction MSE, KL (global means);
                                      # logit-Laplace VAE: device [2] = NLL, image-space MSE (+ KL with the KL term)
        self.loss_parts_format = DALLE_PARTS_FORMAT   # how a training log line shows loss_parts
        self.codebook_usage = None    # VAE with KL: () -> (codes_used, perplexity) of the last batch (a collective)


DALLE_PARTS_FORMAT = " text_ce {:.5f} image_ce {:.5f} z_term {:.3g}"
VAE_PARTS_FORMAT = " recon_mse {:.5f} kl {:.5f}"
VAE_LL_PARTS_FORMAT = " recon_nll {:.5f} recon_mse {:.5f}"
VAE_LL_KL_PARTS_FORMAT = " recon_nll {:.5f} recon_mse {:.5f} kl {:.5f}"


def _to_device(t, dtype, device):
    """Host -> device copy of a step's inputs (pinned host tensors make it asynchronous)."""
    if not torch.is_tensor(t):
        t = torch.as_tensor(t)
    if t.device.type != "cuda":
        t = t.to(device, non_blocking=True)
    if t.dtype != dtype:
        t = t.to(dtype)
    return t.contiguous()


# =====================================================================================================================
# DALL-E
# =====================================================================================================================
def load_vae_model(params, device):
    """src/model_fns.py:35-52: build the (frozen) VAE from params["vae_params"] and locate its checkpoint."""
    vae_params = params.get("vae_params")
    assert vae_params is not None, "vae model config must be supplied"        # model_fns.py:38
    D = params["dataset"]["image_size"]
    vae = build_vae_engine(vae_params, D, device)
    return vae, vae_checkpoint(params)


def vae_checkpoint(params):
    """The VAE checkpoint a DALL-E config names: vae_checkpoint_path, else the latest one under vae_params.model_path
    (None when there is neither)."""
    ckpt = params.get("vae_checkpoint_path")
    if ckpt is None:
        vae_params = params["vae_params"]
        ckpt = latest_checkpoint(vae_params["model_path"]) if vae_params.get("model_path") else None
    return ckpt


DROPOUT_KEYS = ("embed_dropout", "attention_dropout", "residual_dropout")


def dropout_rates(params):
    """(embed, attention, residual) dropout rates of a DALL-E config (src/dalle_mtf/models.py:198, 215, 290, 312, 318);
    a missing or null key is 0.  A rate outside [0, 1) is rejected."""
    rates = []
    for k in DROPOUT_KEYS:
        v = params.get(k)
        r = 0.0 if v is None else float(v)
        if not 0.0 <= r < 1.0:
            raise ValueError(f"{k} = {v!r}: a dropout rate must lie in [0, 1)")
        rates.append(r)
    return tuple(rates)


def attention_layers(params):
    """(attention_types, local_attention_radius) of a DALL-E config.

    local_attention_radius: the reference's key (src/dalle_mtf/models.py:259, default 256), an integer >= 1.
    attention_types: per-layer attention types in GPT-Neo's form, e.g. [[["global", "local"], 3]]: each inner list is
    repeated `count` times and the expansion must give "global", "local", "axial_row", "axial_col" or "conv" (DALL-E's
    row, column and convolutional attention over the image-token grid, DalleEngine), "mlp" (gMLP) or "block_sparse"
    (DeepSpeed-style block-sparse attention) for exactly n_layers layers.  A missing or null key is None: every layer
    global.  Returns the expanded list (or None) and the radius; the kernel size of conv layers is conv_kernel's, the
    layout of block-sparse layers block_sparse_options'."""
    v = params.get("local_attention_radius")
    radius = 256 if v is None else v
    if isinstance(radius, bool) or not isinstance(radius, int) or radius < 1:
        raise ValueError(f"local_attention_radius = {v!r}: must be an integer >= 1")
    spec = params.get("attention_types")
    if spec is None:
        return None, radius
    n_layers = params.get("n_layers")
    types = []
    if not isinstance(spec, (list, tuple)):
        raise ValueError(f"attention_types = {spec!r}: expected a list of [[types...], count] items")
    for item in spec:
        if not (isinstance(item, (list, tuple)) and len(item) == 2 and isinstance(item[0], (list, tuple))
                and isinstance(item[1], int) and not isinstance(item[1], bool) and item[1] >= 1):
            raise ValueError(f"attention_types item {item!r}: expected [[types...], count] with an integer count >= 1")
        for t in item[0]:
            if t not in ATTENTION_TYPES:
                raise ValueError(f"attention_types: unknown attention type {t!r} (expected one of {ATTENTION_TYPES})")
        types += list(item[0]) * item[1]
    if len(types) != n_layers:
        raise ValueError(f"attention_types expands to {len(types)} layers, but n_layers = {n_layers}")
    return types, radius


def activation_function(params):
    """The MLP nonlinearity of a DALL-E config, GPT-Neo's key activation_function: absent, null or "relu" is the
    reference's ReLU, "gelu" mtf's tanh GELU (DalleEngine).  Any other value (other spellings such as "GELU",
    "swish", booleans, numbers) is rejected.  No parameter depends on it, so checkpoints keep their layout."""
    v = params.get("activation_function")
    try:
        return validate_activation("relu" if v is None else v)
    except ValueError:
        raise ValueError(f"activation_function = {v!r}: expected null, \"relu\" or \"gelu\"") from None


def gated_mlp(params):
    """gated_mlp of a DALL-E config: absent, null or false keeps the MLP act(LN2(x) W1 + b1) W2 + b2; true makes it
    DALLE-pytorch's gated FeedForward with the activation_function as the gate's nonlinearity (ReGLU or GEGLU) and W1
    [d, 8d] (DalleEngine).  Only a JSON bool is accepted: 1, "true" or a list is rejected."""
    v = params.get("gated_mlp")
    if v is None:
        return False
    if not isinstance(v, bool):
        raise ValueError(f"gated_mlp = {v!r}: expected null, true or false")
    return v


def sandwich_norm(params):
    """sandwich_norm of a DALL-E config: absent, null or false is off; true normalises each branch output before its
    residual add with a LayerNorm of its own (CogView's Sandwich-LN, DalleEngine), which adds the variables
    layer_i/attn/norm_out/{g,b} and layer_i/mlp/norm_out/{g,b}.  Only a JSON bool is accepted: 1, "true" or a list is
    rejected."""
    v = params.get("sandwich_norm")
    if v is None:
        return False
    if not isinstance(v, bool):
        raise ValueError(f"sandwich_norm = {v!r}: expected null, true or false")
    return validate_sandwich_norm(v)


def layer_scale(params):
    """layer_scale of a DALL-E config: absent, null or false is off (None); true is DALLE-pytorch's LayerScale with its
    initial values by depth (dalle_engine.layer_scale_init); a finite number > 0 is LayerScale starting at that value
    in every layer.  Either adds the variables layer_i/attn/layer_scale (layer_i/gmlp/layer_scale in an 'mlp' layer)
    and layer_i/mlp/layer_scale.  true is never read as the number 1; 0, negative, non-finite, string or list values
    are rejected."""
    return validate_layer_scale(params.get("layer_scale"))


def stable(params):
    """stable of a DALL-E config: absent, null or false is off; true is DALLE-pytorch's stable option (DalleEngine):
    the embedding gradients shrink by 0.1 and the final LayerNorm sees each row divided by its maximum.  It adds no
    variable.  Only a JSON bool is accepted: 1, "true" or a list is rejected."""
    v = params.get("stable")
    if v is None:
        return False
    if not isinstance(v, bool):
        raise ValueError(f"stable = {v!r}: expected null, true or false")
    return validate_stable(v)


def share_input_output_emb(params):
    """share_input_output_emb of a DALL-E config: absent, null or false keeps the output projection
    to_logits/linear_out/kernel; true ties it to the input embedding, logits = hf wte^T + bout (DalleEngine), and the
    checkpoint has no to_logits/linear_out/kernel.  Only a JSON bool is accepted: 1, "true" or a list is rejected."""
    v = params.get("share_input_output_emb")
    if v is None:
        return False
    if not isinstance(v, bool):
        raise ValueError(f"share_input_output_emb = {v!r}: expected null, true or false")
    return validate_share_input_output_emb(v)


def shared_attn_ids(params):
    """shared_attn_ids of a DALL-E config: absent or null gives every layer its own token mixer; a non-empty list of
    integers >= 0, cycled to n_layers, makes the layers with the same id share one (DalleEngine).  The shared module's
    variables are those of its lowest layer.  Returned as given (the engine cycles it); bools, other numbers,
    negative ids and empty lists are rejected."""
    return _shared_ids(params, "shared_attn_ids")


def shared_ff_ids(params):
    """shared_ff_ids of a DALL-E config: as shared_attn_ids, for the MLPs (w1, b1, w2, b2)."""
    return _shared_ids(params, "shared_ff_ids")


def _shared_ids(params, key):
    v = params.get(key)
    if v is None:
        return None
    validate_shared_ids(v, 1, key)
    return list(v)


def shift_tokens(params, image_seq_len=None):
    """shift_tokens of a DALL-E config: absent, null or false is off; true turns on DALLE-pytorch's token shift after
    both LayerNorms of every layer (DalleEngine), which needs a square image-token grid (checked here when
    image_seq_len is given, and by the engine).  Only a JSON bool is accepted: 1, "true" or a list is rejected.  No
    parameter depends on it, so checkpoints keep their layout."""
    v = params.get("shift_tokens")
    if v is None:
        return False
    if not isinstance(v, bool):
        raise ValueError(f"shift_tokens = {v!r}: expected null, true or false")
    return v if image_seq_len is None else validate_shift_tokens(v, image_seq_len)


def conv_kernel(params):
    """conv_attention_kernel of a DALL-E config: the k of "conv" layers' k x k window (DalleEngine), an integer >= 1.
    A missing or null key is 5, DALLE-pytorch's default."""
    v = params.get("conv_attention_kernel")
    try:
        return validate_conv_kernel(5 if v is None else v)
    except ValueError:
        raise ValueError(f"conv_attention_kernel = {v!r}: must be an integer >= 1") from None


def block_sparse_options(params):
    """The DalleEngine keywords of block-sparse layers from a DALL-E config: sparse_block_size (16, 32 or 64; default
    16), sparse_local_window_blocks (an integer >= 1; default 4), sparse_random_blocks (an integer >= 0; a missing or
    null key is DALLE-pytorch's seq_len // block // 4, resolved by the engine) and sparse_layout_seed (an integer >= 0;
    default 0, independent of `seed`).  Any other value raises a ValueError naming the key.  The layout is not stored
    in checkpoints, so sampling must use the training config's keys."""
    keys = ("sparse_block_size", "sparse_local_window_blocks", "sparse_random_blocks", "sparse_layout_seed")
    opts = {k: params.get(k) for k in keys}
    validate_block_sparse(*opts.values(), seq_len=0)
    return opts


def caption_dropout(params):
    """(rate, padding_id) of the config's caption dropout: in mode "train", each sequence's caption is replaced by
    padding_id at every text position with probability `caption_dropout` (a missing or null key is 0), so the model
    also learns p(image | empty caption), the unconditional half of classifier-free guidance.  The rate must lie in
    [0, 1); when it is > 0, padding_id must be an integer in [0, text_vocab_size).  padding_id is None at rate 0."""
    v = params.get("caption_dropout")
    rate = 0.0 if v is None else float(v)
    if not 0.0 <= rate < 1.0:
        raise ValueError(f"caption_dropout = {v!r}: a dropout rate must lie in [0, 1)")
    if rate == 0.0:
        return 0.0, None
    pad, tv = params.get("padding_id"), params.get("text_vocab_size")
    if pad is None or isinstance(pad, bool) or int(pad) != pad or tv is None or not 0 <= pad < tv:
        raise ValueError(f"caption_dropout = {rate} needs padding_id in [0, text_vocab_size = {tv}), got {pad!r}")
    return rate, int(pad)


def input_embedding(params):
    """(image_position_embedding, per_position_padding, padding_id) of a DALL-E config: the DALL-E paper's input
    embedding (extension keys; both absent: the reference's).

    image_position_embedding: absent, null or "absolute" is the reference's learned vector per position (wpe [S, d]);
    "row_col" gives each image token the sum of a row and a column embedding of the W x W token grid, wpe keeping the
    text positions only (DalleEngine).  per_position_padding: absent, null or false is off; true gives every text
    position p its own padding token text_vocab_size + p, used wherever the caption holds padding_id (which must then
    be an integer in [0, text_vocab_size)) and for dropped or unconditional captions.  padding_id is None when it is
    off.  Any other value is rejected."""
    scheme = validate_position_embedding(params.get("image_position_embedding"))
    per_pos = validate_per_position_padding(params.get("per_position_padding"))
    if not per_pos:
        return scheme, False, None
    pad, tv = params.get("padding_id"), params.get("text_vocab_size")
    if pad is None or isinstance(pad, bool) or int(pad) != pad or tv is None or not 0 <= pad < tv:
        raise ValueError(f"per_position_padding needs padding_id in [0, text_vocab_size = {tv}), got {pad!r}")
    return scheme, True, int(pad)


def loss_weights(params):
    """((w_text, w_image) or None, z_loss) of a DALL-E config: the extension keys text_loss_weight / image_loss_weight
    (both or neither; finite reals >= 0 with a sum > 0) and z_loss (a finite real >= 0, default 0).  The loss is then
    (w_t * mean text-row loss + w_i * mean image-row loss) / (w_t + w_i), each row's loss CE + z_loss * lse^2, the
    means over the rows of the global batch (dalle_engine.loss_coefficients)."""
    return validate_loss_weights(params.get("text_loss_weight"), params.get("image_loss_weight"), params.get("z_loss"))


def logits_mask(params):
    """The extension key logits_mask of a DALL-E config (DALLE-pytorch's logits_mask): absent, null or false is the
    reference's objective; true makes text rows (positions p < text_seq_len - 1) normalise over the text ids [0,
    image_offset) only and image rows (image codes and EOS) over [image_offset, V) only (DalleEngine).  Any other value
    is rejected.  Every label must lie in its row's window, which assemble_tokens(_pp) guarantees when the caption ids
    are < text_vocab_size and the VAE codes < image_vocab_size; the loss of a row whose label lies outside is undefined.
    No parameter depends on it, so a checkpoint loads with or without the key."""
    return validate_logits_mask(params.get("logits_mask"))


def rotary_embedding(params, n_embd=None, n_heads=None):
    """(rotary_dim, rotary_base) of a DALL-E config's rotary position embeddings (extension keys; DalleEngine): both
    (None, None) when rotary_dim is absent or null.  rotary_dim must be an even integer with 2 <= rotary_dim <= the
    head dim n_embd / n_heads (taken from params unless given), rotary_base a finite number > 1 (absent or null:
    10000); rotary_base without rotary_dim, and any other value, is rejected.  No parameter depends on them, so
    checkpoints keep their layout."""
    n_embd = params.get("n_embd") if n_embd is None else n_embd
    n_heads = params.get("n_heads") if n_heads is None else n_heads
    count = lambda v: isinstance(v, numbers.Integral) and not isinstance(v, bool)   # noqa: E731
    dh = n_embd // n_heads if count(n_embd) and count(n_heads) and n_heads > 0 else 0
    rot = validate_rotary(params.get("rotary_dim"), params.get("rotary_base"), dh)
    return (None, None) if rot is None else rot


def rotary_emb(params, image_seq_len=None):
    """rotary_emb of a DALL-E config (DALLE-pytorch's rotary embedding, DalleEngine): absent, null or false is off;
    true rotates q, k and v of every attention layer by text / image-row / image-column angles in place of learned
    positions.  Only a JSON bool is accepted; true is refused together with rotary_dim or rotary_base, or with any
    non-null image_position_embedding, and needs a square image-token grid (checked here when image_seq_len is given,
    and by the engine).  A rotary_emb model has no positional_embedding/wpe variable."""
    v = params.get("rotary_emb")
    rot = (params.get("rotary_dim"), params.get("rotary_base"))
    on = validate_rotary_emb(v, 1 if image_seq_len is None else image_seq_len,
                             None if rot == (None, None) else rot, params.get("image_position_embedding"))
    return on


def dalle_model_fn(features, labels, mode, params):
    """src/model_fns.py:55-236.  features: images f32 [B,H,W,C] in [-1,1] (NHWC); labels: caption ids i32
    [B, text_seq_len].  (The reference's own comment has them swapped; the code uses them this way.)"""
    mode_str = mode_to_str(mode)
    if mode == PREDICT:
        raise NotImplementedError                                             # model_fns.py:135-136
    cap_rate, pad_id = caption_dropout(params)
    attention_types, local_radius = attention_layers(params)
    conv_k = conv_kernel(params)
    sparse = block_sparse_options(params)
    weights, z_loss = loss_weights(params)
    pos_scheme, per_pos, pp_pad = input_embedding(params)
    activation = activation_function(params)
    gated = gated_mlp(params)
    shift = shift_tokens(params)
    sandwich = sandwich_norm(params)
    scale = layer_scale(params)
    stab = stable(params)
    tied = share_input_output_emb(params)
    attn_ids, ff_ids = shared_attn_ids(params), shared_ff_ids(params)
    mask = logits_mask(params)
    rotary_dim, rotary_base = rotary_embedding(params)
    # rotary_emb needs a square grid: checked here from the VAE config, before anything reaches the device
    rot_emb = rotary_emb(params)
    if rot_emb:
        rotary_emb(params, vae_grid_size(params["vae_params"], params["dataset"]["image_size"]) ** 2)
    L.require_device()
    dp = params.get("_dp") or DataParallel().init()
    device = torch.device("cuda", torch.cuda.current_device())
    mesh, _ = parse_mesh(params["mesh_shape"], params["layout"])            # model_fns.py:81-82
    if mesh.get("model", 1) != 1 and dp.rank == 0:
        print(f"note: mesh axis model:{mesh['model']} has no layout rule in the reference either (pure replication); "
              f"this engine runs data:{dp.world} and does not duplicate work")

    # ---- frozen VAE tokenizer (model_fns.py:63-77)
    vae, vae_ckpt = load_vae_model(params, device)
    if vae_ckpt is not None:
        state = load_checkpoint(local_path(vae_ckpt))
        vae.load_params({k[len("vae/"):]: v for k, v in state.items() if k.startswith("vae/")})
    elif params.get("vae_random_init"):
        vae.init_params(seed=params.get("vae_seed") or 0)   # extension key: throughput runs without a checkpoint
    else:
        raise AssertionError("pretrained vae needed for training")              # model_fns.py:41
    image_seq_len = vae.image_seq_len                                           # model_fns.py:68
    global_batch = params[f"{mode_str}_batch_size"]                             # model_fns.py:69
    first_row, local_batch = dp.shard(global_batch)
    rates = dropout_rates(params)

    model = DalleEngine(n_embd=params["n_embd"], n_layers=params["n_layers"], n_heads=params["n_heads"],
                        text_vocab_size=params["text_vocab_size"], image_vocab_size=params["image_vocab_size"],
                        text_seq_len=params["text_seq_len"], image_seq_len=image_seq_len, device=device,
                        recompute_grad=bool(params.get("recompute_grad")) and mode == TRAIN,   # models.py:342
                        # extension key: shard fp32 master + Adam slots across the data-parallel ranks (ZeRO-1) —
                        # what lets the d = 4096 configuration fit 80 GB GPUs in pure data parallelism
                        zero=dp if (params.get("optimizer_state_sharding") and dp.enabled) else None,
                        dropout=rates, dropout_seed=params.get("seed") or 0,
                        attention_types=attention_types, local_attention_radius=local_radius,  # models.py:229-301
                        conv_attention_kernel=conv_k, loss_weights=weights, z_loss=z_loss,
                        image_position_embedding=None if rot_emb else pos_scheme, per_position_padding=per_pos,
                        activation=activation, logits_mask=mask, rotary_dim=rotary_dim, rotary_base=rotary_base,
                        gated_mlp=gated, shift_tokens=shift, sandwich_norm=sandwich, layer_scale=scale,
                        stable=stab, share_input_output_emb=tied, shared_attn_ids=attn_ids, shared_ff_ids=ff_ids,
                        rotary_emb=rot_emb, **sparse)
    if params["bf_16"] is False and dp.rank == 0:
        print("note: bf_16=false — the engine still runs activations and matmul operands in bf16 with fp32 "
              "accumulation, fp32 master weights / optimiser state (there is no fp32 tensor-core path yet)")
    if vae.K > params["image_vocab_size"]:
        raise ValueError(f"vae num_tokens {vae.K} exceeds image_vocab_size {params['image_vocab_size']}: image ids "
                         "would index past the embedding table (SURVEY.md Appendix C.4)")
    model.init_params(seed=params.get("seed") or 0)
    if dp.rank == 0:
        print_n_params(model.n_params())                                        # get_graph_info, model_fns.py:186

    S = model.S
    tokens = torch.empty(local_batch, S, dtype=torch.int32, device=device)
    total_tokens_global = global_batch * S
    # micro-batching (model_fns.py:144-166): tokens_per_mb_per_replica -> number of sequential micro-batches
    tpmb = params.get("tokens_per_mb_per_replica")
    num_microbatches = 1
    if mode == TRAIN and tpmb:
        seqs_per_mb = max(1, int(tpmb) // S)
        num_microbatches = max(1, -(-local_batch // seqs_per_mb))
        while local_batch % num_microbatches:
            num_microbatches += 1
    params["num_microbatches"] = num_microbatches                               # model_fns.py:154
    opt = OptimizerConfig(params) if mode == TRAIN else None
    spec = StepSpec(mode, model, dp=dp, extra={"vae": vae})

    def assemble(features, labels, caption_drop=None):
        img = _to_device(features, torch.float32, device).view(local_batch, vae.img_H, vae.img_W, vae.img_C)
        text = _to_device(labels, torch.int32, device).view(local_batch, params["text_seq_len"])
        img_ids = vae.encode_tokens(img)                                        # model_fns.py:72-77
        if per_pos:   # padding ids (and dropped captions) become the per-position pads
            ops.assemble_tokens_pp(text, img_ids, tokens, model.image_offset, pp_pad, model.pad_base,
                                   caption_drop=caption_drop)
        else:
            ops.assemble_tokens(text, img_ids, tokens, model.text_vocab_size,   # model_fns.py:117-122
                                caption_drop=caption_drop, pad_id=pad_id)
        return tokens

    def loss_value():
        # sum of per-token losses over all ranks (all-reduced with the gradients) / global token count
        return model.grads[model.aux_off:model.aux_off + 1]

    # weighted loss: the coefficients depend on the global batch only (not on the rank count, the micro-batch size or a
    # resume), aux slot 0 holds the loss itself and slots 1-3 the sums the parts are formed from
    weighted = model.weighted_loss
    loss_scale = 1.0 if weighted else 1.0 / total_tokens_global
    part_scales = torch.tensor(model.loss_part_scales(global_batch), dtype=torch.float32, device=device) \
        if weighted else None

    def loss_parts(sums):
        return sums[1:4] * part_scales if weighted else None

    dp.hint_tokens_per_gpu(local_batch * S)

    def train_op(features, labels):
        # caption dropout of the global step, one decision per global sequence index, drawn for the whole local batch
        # before micro-batching: the same captions drop whatever the rank count, micro-batch size or resume point
        # (labels are shifted from these tokens, so a dropped caption is dropped from the targets too)
        cap = L.make_dropout(cap_rate, params.get("seed") or 0, spec.global_step, L.SITE_CAPTION, first_row) \
            if cap_rate else None
        toks = assemble(features, labels, cap)
        model.zero_grads()
        mb = local_batch // num_microbatches
        hook = dp.make_bucket_hook(model.grads)
        for i in range(num_microbatches):
            # dropout masks of the global step, indexed by the global sequence index of each row: the same masks
            # whatever the rank count or micro-batch size (models.py:198-323 apply them in mode "train" only)
            model.forward(toks[i * mb:(i + 1) * mb], step=spec.global_step, row0=first_row + i * mb,
                          global_batch=global_batch)
            last = i == num_microbatches - 1
            if last:
                dp.begin_overlap()
            # loss = mean over the GLOBAL batch (models.py:353-354): every rank back-props local_sum / (B*S) and the
            # all-reduce SUMs the shard partials (mtf semantics, SURVEY.md §8e); the weighted loss carries its global
            # normalisation in its coefficients
            model.backward(1.0 if weighted else 1.0 / total_tokens_global, on_bucket_ready=hook if last else None)
        dp.wait()
        lr = opt.learning_rate(spec.global_step)                                # step counter before the increment
        model.optimizer_step(lr, beta1=opt.beta_1, beta2=opt.beta_2, eps=opt.epsilon,
                             weight_decay=opt.weight_decay, clip=opt.gradient_clipping)
        spec.global_step += 1                                                   # model_fns.py:201
        spec.lr = lr
        spec.loss_sum = loss_value()
        spec.loss_scale = loss_scale
        spec.loss_parts = loss_parts(model.grads[model.aux_off:model.aux_off + 4])
        return spec.loss_sum

    def eval_op(features, labels):
        toks = assemble(features, labels)
        acc = torch.zeros(4 if weighted else 1, dtype=torch.float32, device=device)
        model.forward(toks, loss_accum=acc, global_batch=global_batch)
        dp.all_reduce_now(acc)
        spec.loss_sum, spec.loss_scale = acc[:1], loss_scale
        spec.loss_parts = loss_parts(acc)
        return spec.loss_sum

    def state_fn():
        st = {k: v for k, v in model.export_params().items()}
        if model.zero is not None:      # sharded Adam slots are not gathered into rank 0's checkpoint (throughput config)
            st["global_step"] = spec.global_step
            return st
        st.update({k + "/adam_m": v for k, v in model.export_params(model.adam_m).items()})   # optimizers.py:139
        st.update({k + "/adam_v": v for k, v in model.export_params(model.adam_v).items()})   # optimizers.py:147
        st["global_step"] = spec.global_step
        return st

    def load_fn(st):
        names = [k for k in st if not k.endswith("/adam_m") and not k.endswith("/adam_v") and k != "global_step"]
        if model.zero is not None and mode == TRAIN:
            # restarting Adam's moments from zero at the full learning rate would silently change the run
            raise L.DB200Error("optimizer_state_sharding: ZeRO-1 checkpoints hold no Adam slots (DESIGN.md §7) and "
                               "resuming training needs them; such a checkpoint can be evaluated, exported or sampled")
        model.load_params({k: st[k] for k in names})                                # master + bf16 shadow
        if model.zero is not None:      # evaluation: the parameters are all it needs
            spec.global_step = int(st.get("global_step", 0))
            return
        for suffix, flat in (("/adam_m", model.adam_m), ("/adam_v", model.adam_v)):
            model.load_flat(flat, {k: st[k + suffix] for k in names})
        spec.global_step = int(st.get("global_step", 0))

    spec.train_op = train_op if mode == TRAIN else None
    spec.eval_op = eval_op
    spec.state_fn, spec.load_fn = state_fn, load_fn
    spec.tokens_per_step = total_tokens_global
    spec.assemble = assemble
    return spec


# =====================================================================================================================
# discrete VAE
# =====================================================================================================================
def vae_temperature(step, params):
    """src/model_fns_tf.py:40-45."""
    if params.get("temp_anneal_steps"):
        frac = min(step / params["temp_anneal_steps"], 1.0)
        return params["temp_start"] - frac * (params["temp_start"] - params["temp"])
    t = params.get("temp")
    return 1.0 if t is None else t


def validate_kl_weight(beta, anneal_steps=None):
    """(beta, anneal_steps) of the VAE's KL term, or (None, None) without one.  beta: a finite real >= 0 (not a bool);
    anneal_steps: None or an integer >= 1 (not a bool), only together with beta."""
    if beta is None:
        if anneal_steps is not None:
            raise ValueError(f"kl_anneal_steps = {anneal_steps!r} without kl_loss_weight has no effect")
        return None, None
    if isinstance(beta, bool) or not isinstance(beta, numbers.Real) or not math.isfinite(beta) or beta < 0:
        raise ValueError(f"kl_loss_weight = {beta!r}: must be a finite real >= 0")
    if anneal_steps is not None and (isinstance(anneal_steps, bool) or not isinstance(anneal_steps, numbers.Integral)
                                     or anneal_steps < 1):
        raise ValueError(f"kl_anneal_steps = {anneal_steps!r}: must be an integer >= 1")
    return float(beta), None if anneal_steps is None else int(anneal_steps)


def kl_loss_weight(params):
    """(beta, anneal_steps) of a VAE config's extension keys kl_loss_weight / kl_anneal_steps (validate_kl_weight).
    The objective is then MSE + beta_t * KL, KL the mean over the latent rows of the global batch of
    KL(softmax(logits) || Uniform(K)), beta_t = vae_kl_weight(step, params)."""
    return validate_kl_weight(params.get("kl_loss_weight"), params.get("kl_anneal_steps"))


def vae_kl_weight(step, params):
    """beta_t of the KL term at global step `step`: beta * min(step / kl_anneal_steps, 1), or beta without the anneal
    key (None without kl_loss_weight).  A function of the step alone, so a resumed run continues the schedule."""
    beta, anneal = kl_loss_weight(params)
    if beta is None:
        return None
    return beta * min(step / anneal, 1.0) if anneal else beta


def reconstruction_loss(value):
    """The VAE's reconstruction term from its config key reconstruction_loss (an extension): None (absent, null) or
    "mse" is the reference's MSE, "logit_laplace" the DALL-E paper's logit-Laplace NLL; anything else is rejected."""
    if value is None:
        return "mse"
    if not isinstance(value, str) or value not in RECONSTRUCTION_LOSSES:
        raise ValueError(f"reconstruction_loss = {value!r}: must be one of {RECONSTRUCTION_LOSSES} (or null)")
    return value


VAE_ARCHITECTURES = ("reference", "dalle_paper", "vqgan")
VQGAN_KEYS = ("ch", "ch_mult", "num_res_blocks", "attn_resolutions", "z_channels", "embed_dim", "resolution")
PAPER_VAE_DEFAULTS = {"n_hid": 256, "n_blk_per_group": 2, "group_count": 4, "n_init": 128}


def vae_architecture(params, image_size):
    """The network of a VAE config: None for the reference's (key architecture absent, null or "reference"), else the
    geometry dict {n_hid, n_blk_per_group, group_count, n_init} of the DALL-E paper's ("dalle_paper"; absent keys
    take PAPER_VAE_DEFAULTS).  Raises ValueError for any other architecture, for convblocks or stack_factor > 1 with
    the paper's network, and for a geometry it does not define (PaperVaeEngine)."""
    arch = params.get("architecture")
    if arch is None or arch == "reference":
        return None
    if arch == "vqgan":
        return vqgan_geometry(params, image_size)
    if arch != "dalle_paper":
        raise ValueError(f"architecture = {arch!r}: must be one of {VAE_ARCHITECTURES} (or null)")
    if params.get("convblocks") is not None:
        raise ValueError("convblocks describes the reference network; architecture \"dalle_paper\" is sized by n_hid, "
                         "n_blk_per_group, group_count and n_init")
    sf = params.get("stack_factor")
    if sf is not None and sf != 1:
        raise ValueError(f"stack_factor = {sf!r}: architecture \"dalle_paper\" takes no stack_factor > 1")
    geo = {k: (d if params.get(k) is None else params[k]) for k, d in PAPER_VAE_DEFAULTS.items()}
    check_paper_geometry(image_size, **geo)
    return geo


def vqgan_geometry(params, image_size):
    """The geometry of a VAE config with architecture "vqgan" (taming's ddconfig key names; num_tokens is taming's
    n_embed): {ch, ch_mult, num_res_blocks, attn_resolutions, z_channels, embed_dim, resolution, quantizer}, quantizer
    "vq" (taming's VectorQuantizer, the default) or "gumbel" (its GumbelQuantize).  Raises ValueError,
    naming the key, for a missing key, for keys of the other networks, for use_bf16 false (the tokenizer runs bf16
    activations only) and for a geometry the kernels do not cover."""
    for k in ("convblocks", "n_hid", "n_blk_per_group", "group_count", "n_init"):
        if params.get(k) is not None:
            raise ValueError(f"{k} sizes another network; architecture \"vqgan\" is sized by taming's keys "
                             f"{VQGAN_KEYS}")
    sf = params.get("stack_factor")
    if sf is not None and sf != 1:
        raise ValueError(f"stack_factor = {sf!r}: architecture \"vqgan\" takes no stack_factor > 1")
    if params.get("use_bf16") is False:
        raise ValueError("use_bf16 = false: architecture \"vqgan\" runs bf16 activations only (DESIGN.md §4)")
    for k in ("reconstruction_loss", "kl_loss_weight"):
        if params.get(k) is not None:
            raise ValueError(f"{k}: a VQGAN tokenizer is used frozen and has no training objective here")
    missing = [k for k in VQGAN_KEYS + ("num_tokens",) if params.get(k) is None]
    if missing:
        raise ValueError(f"{missing[0]}: missing from the architecture \"vqgan\" config (keys: {VQGAN_KEYS})")
    geo = {k: params[k] for k in VQGAN_KEYS}
    geo["quantizer"] = "vq" if params.get("quantizer") is None else params["quantizer"]
    check_vqgan_geometry(image_size, num_tokens=params["num_tokens"], **geo)
    return geo


def vae_grid_size(params, image_size):
    """Side of a VAE config's token grid: image_size / 2^(len(ch_mult) - 1) for a VQGAN, image_size /
    2^(group_count - 1) for the paper's network, image_size / stack_factor / 2^len(convblocks) for the reference's."""
    geo = vae_architecture(params, image_size)
    if params.get("architecture") == "vqgan":
        return image_size // 2 ** (len(geo["ch_mult"]) - 1)
    if geo is not None:
        return image_size // 2 ** (geo["group_count"] - 1)
    convblocks = params.get("convblocks") or [(3, 64), (3, 128), (3, 256)]
    return image_size // (params.get("stack_factor") or 1) // (2 ** len(convblocks))


def build_vae_engine(params, image_size, device, kl=False):
    """The VAE engine of a VAE config (vae_architecture picks the network)."""
    recon = reconstruction_loss(params.get("reconstruction_loss"))
    geo = vae_architecture(params, image_size)
    if params.get("architecture") == "vqgan":
        return VqganEngine(num_tokens=params["num_tokens"], image_size=image_size,
                           input_channels=params.get("input_channels") or 3, device=device, **geo)
    if geo is not None:
        return PaperVaeEngine(num_tokens=params["num_tokens"], image_size=image_size,
                              input_channels=params.get("input_channels") or 3, use_bf16=bool(params.get("use_bf16")),
                              recompute_grad=bool(params.get("recompute_grad")), device=device, kl=kl,
                              reconstruction_loss=recon, **geo)
    return VaeEngine(num_tokens=params["num_tokens"], image_size=image_size,
                     convblocks=params.get("convblocks") or [(3, 64), (3, 128), (3, 256)],
                     input_channels=params.get("input_channels") or 3,
                     recompute_grad=bool(params.get("recompute_grad")),
                     use_bf16=bool(params.get("use_bf16")),   # bf16 -> wgmma implicit-GEMM convolutions
                     stack_factor=params.get("stack_factor") or 1, device=device, kl=kl, reconstruction_loss=recon)


def vae_model_fn(features, labels, mode, params):
    """src/model_fns_tf.py:9-114.  features = labels = images f32 [B,H,W,C] in [-1,1].

    With the extension key kl_loss_weight (and optionally kl_anneal_steps), spec.loss_sum * spec.loss_scale is the
    objective MSE + beta_t * KL, spec.loss_parts the device [2] (MSE, KL) of the global batch and
    spec.codebook_usage() the (codes_used, perplexity) of its first-maximum codes.

    With reconstruction_loss "logit_laplace" the reconstruction term is the mean logit-Laplace NLL and spec.loss_parts
    the device (NLL, image-space MSE) or, with the KL term, (NLL, image-space MSE, KL)."""
    mode_str = mode_to_str(mode)
    if mode == PREDICT:
        raise NotImplementedError                                             # model_fns_tf.py:29-30
    kl_beta, _ = kl_loss_weight(params)
    kl_on = kl_beta is not None
    recon_loss = reconstruction_loss(params.get("reconstruction_loss"))
    ll = recon_loss == "logit_laplace"
    if params.get("architecture") == "vqgan":
        raise ValueError("architecture = \"vqgan\": a VQGAN is imported from taming-transformers "
                         "(tools/import_vqgan.py), not trained here (that needs LPIPS weights and a discriminator)")
    vae_architecture(params, params["dataset"]["image_size"])   # rejects an invalid network before any device work
    n_aux = 3 if ll else (2 if kl_on else 1)    # aux slots: [recon term, KL, image-space MSE]
    L.require_device()
    dp = params.get("_dp") or DataParallel().init()
    device = torch.device("cuda", torch.cuda.current_device())
    H = params["dataset"]["image_size"]                                       # model_fns_tf.py:13
    global_batch = params[f"{mode_str}_batch_size"]
    _, local_batch = dp.shard(global_batch)
    model = build_vae_engine(params, H, device, kl=kl_on)
    model.init_params(seed=params.get("seed") or 0)
    if dp.rank == 0:
        print_n_params(model.n_params())
        if params.get("recompute_grad"):
            print("note: recompute_grad=true (src/vae_tf/models.py:8-43) — the engine keeps the residual-pair "
                  "activations instead of recomputing them (they fit in HBM many times over); gradients are identical")
    tg = params.get("train_gumbel_hard")
    eg = params.get("eval_gumbel_hard")
    train_gumbel = True if tg is None else tg                                 # model_fns_tf.py:32
    eval_gumbel = True if eg is None else eg                                  # model_fns_tf.py:33
    hard = train_gumbel if mode == TRAIN else eval_gumbel
    rows = local_batch * model.hw * model.hw
    noise = torch.empty(rows, model.K, dtype=torch.float32, device=device)
    gen = torch.Generator(device=device).manual_seed(1234 + dp.rank)
    spec = StepSpec(mode, model, dp=dp)
    n_global = global_batch * H * H * model.img_C

    def draw_noise():
        # tf.random_uniform(minval=1e-9, maxval=1.) (src/vae_tf/layers.py:8-13); RNG stream is ours (SURVEY §7)
        noise.uniform_(1e-9, 1.0, generator=gen)
        return noise

    def run(features, train):
        img = _to_device(features, torch.float32, device).view(local_batch, H, H, model.img_C)
        temp = vae_temperature(spec.global_step, params)
        spec.kl_weight = vae_kl_weight(spec.global_step, params)
        u = params.get("_gumbel_u")
        u = draw_noise() if u is None else u
        model.zero_grads()
        # adds sum((img-out)^2)/local_numel (logit-Laplace: the mean NLL) into aux slot 0, with the KL term the local
        # mean KL into slot 1, and with logit-Laplace the image-space MSE into slot 2
        recon = model.forward(img, u, temp, hard, kl_weight=spec.kl_weight)
        return recon

    def report(sums):
        # sums: the all-reduced aux slots [recon term, KL, image-space MSE], each the SUM over ranks of the local means
        if ll:
            parts = [sums[:1], sums[2:3]] + ([sums[1:2]] if kl_on else [])
            spec.loss_parts = torch.cat(parts) * (1.0 / dp.world)
            spec.loss_sum = sums[:1] + spec.kl_weight * sums[1:2] if kl_on else sums[:1]
            spec.loss_scale = 1.0 / dp.world
        elif kl_on:
            spec.loss_parts = sums[:2] * (1.0 / dp.world)
            spec.loss_sum, spec.loss_scale = sums[:1] + spec.kl_weight * sums[1:2], 1.0 / dp.world
        else:
            spec.loss_sum, spec.loss_scale = sums[:1], 1.0 / dp.world

    def usage():
        # code counts of the global batch: one all-reduce, only when asked (every rank must ask)
        counts = model.code_counts().to(torch.float32)
        dp.all_reduce_now(counts)
        return codebook_usage(counts)

    def train_op(features, labels=None):
        run(features, True)
        # CrossShardOptimizer: cross-replica MEAN of the gradients (model_fns_tf.py:61) = bucketed SUM all-reduce that
        # overlaps with the rest of backward (decoder, codebook, encoder ranges), then 1/N inside the Adam kernel
        dp.begin_overlap()
        model.backward(on_bucket_ready=dp.make_bucket_hook(model.grads))
        dp.wait()
        spec.global_step += 1
        model.optimizer_step(params["lr"], spec.global_step, grad_scale=1.0 / dp.world)   # model_fns_tf.py:58-60
        # each rank's aux slots hold its local means, all-reduced with the decoder bucket; the SUM over ranks / N
        report(model.grads[model.aux_off:model.aux_off + n_aux])
        return spec.loss_sum

    def eval_op(features, labels=None):
        run(features, False)
        acc = model.grads[model.aux_off:model.aux_off + n_aux].clone()
        dp.all_reduce_now(acc)
        report(acc)
        return spec.loss_sum

    def state_fn():
        st = {"vae/" + k: v for k, v in model.export_params().items()}
        st.update({"vae/" + k + "/Adam": v for k, v in model.export_params(model.adam_m).items()})
        st.update({"vae/" + k + "/Adam_1": v for k, v in model.export_params(model.adam_v).items()})
        st["global_step"] = spec.global_step
        return st

    def load_fn(st):
        # master weights (+ the bf16 shadow / split codebook derived from them), then the Adam slots straight into
        # their flat buffers: the compute copies must never be refreshed from anything but the weights
        model.load_params({k[len("vae/"):]: v for k, v in st.items()
                           if k.startswith("vae/") and not k.endswith("/Adam") and not k.endswith("/Adam_1")})
        for suffix, flat in (("/Adam", model.adam_m), ("/Adam_1", model.adam_v)):
            model.load_flat(flat, {k[len("vae/"):-len(suffix)]: v for k, v in st.items() if k.endswith(suffix)})
        spec.global_step = int(st.get("global_step", 0))

    spec.train_op = train_op if mode == TRAIN else None
    spec.eval_op = eval_op
    spec.state_fn, spec.load_fn = state_fn, load_fn
    spec.images_per_step = global_batch
    spec.n_global = n_global
    spec.kl_weight = None
    if kl_on:
        spec.loss_parts_format = VAE_PARTS_FORMAT
        spec.codebook_usage = usage
    if ll:
        spec.loss_parts_format = VAE_LL_KL_PARTS_FORMAT if kl_on else VAE_LL_PARTS_FORMAT
    return spec
