"""DALL-E transformer training engine on the sm_90a kernels (host side: buffer plan + kernel sequencing).

Mirrors what the reference builds as an mtf graph in src/dalle_mtf/models.py:141-416 and differentiates with
mtf.gradients (src/optimizers.py:34): here forward and backward are explicit kernel sequences over pre-allocated
buffers.  PyTorch owns the memory; all arithmetic is in libdalle_b200.so.

HBM layout
  * parameters, gradients, Adam m / v: ONE flat fp32 buffer each, same offsets (``ParamLayout``), plus a flat bf16
    "shadow" copy of the parameters that the GEMMs / gather read (mtf VariableDType: slice fp32 -> activation bf16,
    src/dalle_mtf/ops.py:76-82).  Order = forward order, so backward finishes gradients from the END of the buffer
    towards the front and contiguous tail ranges can be all-reduced while backward is still running.
  * q|k|v kernels are stored fused as one [d, 3d] matrix (columns q, k, v), the vocabulary projection as
    [d, Vpad] with Vpad = V rounded up to 64 (TMA needs 16-byte row pitch; pad columns stay exactly zero).
  * activations bf16 [T = B*S, features]; per-layer intermediates are kept for backward unless recompute_grad.
"""
import math
import numbers

import torch

from . import lib as L
from . import ops

BF16, F32, I32 = torch.bfloat16, torch.float32, torch.int32


def _round_up(x, m):
    return (x + m - 1) // m * m


class ParamLayout:
    """name -> (offset, shape) inside the flat buffers.  Every offset is a multiple of 64 elements.  An alias (a shared
    module's name in a layer that does not own it) has its owner's entry but no place in `order` and no size."""

    def __init__(self):
        self.entries = {}
        self.order = []
        self.aliases = {}
        self.size = 0

    def add(self, name, shape):
        n = 1
        for s in shape:
            n *= s
        self.entries[name] = (self.size, tuple(shape))
        self.order.append(name)
        self.size += _round_up(n, 64)

    def alias(self, name, owner):
        """Make `name` a second name of the existing entry `owner` (same offset, same storage)."""
        self.entries[name] = self.entries[owner]
        self.aliases[name] = owner

    def view(self, flat, name):
        off, shape = self.entries[name]
        n = 1
        for s in shape:
            n *= s
        return flat[off:off + n].view(*shape)

    def span(self, first, last):
        """[start, end) element range covering entries first..last (inclusive, in layout order)."""
        o0, _ = self.entries[first]
        o1, shp = self.entries[last]
        n = 1
        for s in shp:
            n *= s
        return o0, o1 + _round_up(n, 64)


ATTN_MODULE = ("wqkv", "wo", "o_b")                 # an attention layer's token mixer
GMLP_MODULE = ("gm_win", "gm_bin", "sgu_g", "sgu_b", "sgu_w", "sgu_c", "gm_wout", "gm_bout")   # a gMLP layer's
FF_MODULE = ("w1", "b1", "w2", "b2")                 # the MLP


def param_layout(d, n_layers, V, S, text_len=None, grid_w=None, gated_mlp=False, sandwich_norm=False, mlp_layers=None,
                 layer_scale=False, tied=False, attn_owner=None, ff_owner=None, wpe=True):
    """The flat-buffer layout of a DalleEngine of width d, n_layers blocks, vocabulary V (EOS included) and sequence
    length S: forward order, the vocabulary projection and its bias padded to a multiple of 64 columns.  grid_w (row /
    column image positions, S = text_len + grid_w^2): wpe holds the text_len text positions and image_row / image_col
    the grid_w rows and columns of the image-token grid.  gated_mlp: w1 is [d, 8d] and b1 [8d], the value columns
    first and the gate columns second.  sandwich_norm: each layer ends with its two output LayerNorms, lna_g / lna_b
    (attention branch) and lnm_g / lnm_b (MLP branch), inside the layer's span l{i}.ln1_g .. layer_last(i).
    mlp_layers: per layer, True for a gMLP token-mixing layer, whose gm_win [d, 4d], gm_bin [4d], sgu_g / sgu_b [2d],
    sgu_w [S, S], sgu_c [S], gm_wout [2d, d] and gm_bout [d] take the place of wqkv, wo and o_b.  layer_scale: each
    layer ends with its two LayerScale vectors, lsa (the token mixer's branch) and lsm (the MLP's), after the sandwich
    LayerNorms.
    tied (share_input_output_emb): wte is [Vpad, d], its pad rows exactly zero, and is also the vocabulary projection;
    there is no wout.  attn_owner / ff_owner (shared_attn_ids / shared_ff_ids): per layer, the layer whose token mixer
    (ATTN_MODULE or GMLP_MODULE) / MLP (FF_MODULE) it uses.  A layer that is not its module's owner gets aliases of the
    owner's entries, so that layer i's own entries still run contiguously from l{i}.ln1_g.
    wpe False (rotary_emb): no learned position embedding; wte is followed by the first layer."""
    w1_cols = 8 * d if gated_mlp else 4 * d
    Vpad = _round_up(V, 64)
    attn_owner = list(range(n_layers)) if attn_owner is None else attn_owner
    ff_owner = list(range(n_layers)) if ff_owner is None else ff_owner
    lay = ParamLayout()
    lay.add("wte", (Vpad if tied else V, d))
    if grid_w is None:
        if wpe:
            lay.add("wpe", (S, d))
    else:
        lay.add("wpe", (text_len, d))
        lay.add("image_row", (grid_w, d)); lay.add("image_col", (grid_w, d))

    def module(i, owner, names, add):
        if owner[i] == i:
            return add()
        for k in names:
            lay.alias(f"l{i}.{k}", f"l{owner[i]}.{k}")

    for i in range(n_layers):
        p = f"l{i}."
        lay.add(p + "ln1_g", (d,)); lay.add(p + "ln1_b", (d,))
        if mlp_layers is not None and mlp_layers[i]:
            module(i, attn_owner, GMLP_MODULE, lambda: (
                lay.add(p + "gm_win", (d, 4 * d)), lay.add(p + "gm_bin", (4 * d,)),
                lay.add(p + "sgu_g", (2 * d,)), lay.add(p + "sgu_b", (2 * d,)),
                lay.add(p + "sgu_w", (S, S)), lay.add(p + "sgu_c", (S,)),
                lay.add(p + "gm_wout", (2 * d, d)), lay.add(p + "gm_bout", (d,))))
        else:
            module(i, attn_owner, ATTN_MODULE, lambda: (
                lay.add(p + "wqkv", (d, 3 * d)), lay.add(p + "wo", (d, d)), lay.add(p + "o_b", (d,))))
        lay.add(p + "ln2_g", (d,)); lay.add(p + "ln2_b", (d,))
        module(i, ff_owner, FF_MODULE, lambda: (
            lay.add(p + "w1", (d, w1_cols)), lay.add(p + "b1", (w1_cols,)),
            lay.add(p + "w2", (4 * d, d)), lay.add(p + "b2", (d,))))
        if sandwich_norm:
            lay.add(p + "lna_g", (d,)); lay.add(p + "lna_b", (d,))
            lay.add(p + "lnm_g", (d,)); lay.add(p + "lnm_b", (d,))
        if layer_scale:
            lay.add(p + "lsa", (d,)); lay.add(p + "lsm", (d,))
    lay.add("lnf_g", (d,)); lay.add("lnf_b", (d,))
    if not tied:
        lay.add("wout", (d, Vpad))
    lay.add("bout", (Vpad,))
    return lay


ATTENTION_TYPES = ("global", "local", "axial_row", "axial_col", "conv", "mlp", "block_sparse")
AXIAL_AXIS = {"axial_row": 0, "axial_col": 1}


def layer_radii(attention_types, radius, n_layers):
    """Per-layer attention radius: None for a "global" (or axial, or conv) layer, `radius` for a "local" one (attention_types
    None: every layer global)."""
    if isinstance(radius, bool) or not isinstance(radius, numbers.Integral) or radius < 1:
        raise ValueError(f"local_attention_radius must be an integer >= 1, got {radius!r}")
    if attention_types is None:
        return [None] * n_layers
    types = list(attention_types)
    if len(types) != n_layers or any(t not in ATTENTION_TYPES for t in types):
        raise ValueError(f"attention_types must list one of {ATTENTION_TYPES} for each of the {n_layers} layers, got "
                         f"{attention_types!r}")
    return [int(radius) if t == "local" else None for t in types]


def layer_mlp(attention_types, n_layers, seq_len, n_embd):
    """Per-layer flag of the gMLP token-mixing layers ("mlp"), refusing a geometry their kernels cannot run: the
    sequence length must be a multiple of 64 (tile-aligned per-sequence rows for TMA) and 2 n_embd, the width of the
    spatial gating unit's LayerNorm, one of LAYERNORM_WIDTHS."""
    if attention_types is None:
        return [False] * n_layers
    flags = [t == "mlp" for t in attention_types]
    if any(flags):
        if seq_len % 64:
            raise L.DB200Error(f"attention_types 'mlp': text_seq_len + image_seq_len = {seq_len} must be a multiple of "
                               "64")
        if 2 * n_embd not in LAYERNORM_WIDTHS:
            raise L.DB200Error(f"attention_types 'mlp': n_embd {n_embd} gives a spatial gating unit of width "
                               f"{2 * n_embd}, which the LayerNorm kernels do not implement (one of {LAYERNORM_WIDTHS})")
    return flags


def layer_axial(attention_types, text_seq_len, image_seq_len, n_layers):
    """Per-layer axial geometry: (text_seq_len, W, axis) for an "axial_row" (axis 0) or "axial_col" (axis 1) layer,
    where the image tokens form a W x W grid (image_seq_len = W^2), and None for any other layer."""
    if attention_types is None:
        return [None] * n_layers
    types = list(attention_types)
    if not any(t in AXIAL_AXIS for t in types):
        return [None] * len(types)
    W = math.isqrt(image_seq_len)
    if W * W != image_seq_len:
        raise ValueError(f"axial attention layers need a square image-token grid, but image_seq_len = {image_seq_len} "
                         "is not a square")
    return [(int(text_seq_len), W, AXIAL_AXIS[t]) if t in AXIAL_AXIS else None for t in types]


def validate_conv_kernel(kernel):
    """The kernel size of convolutional attention layers: an integer >= 1."""
    if isinstance(kernel, bool) or not isinstance(kernel, numbers.Integral) or kernel < 1:
        raise ValueError(f"conv_attention_kernel must be an integer >= 1, got {kernel!r}")
    return int(kernel)


def layer_conv(attention_types, text_seq_len, image_seq_len, kernel, n_layers):
    """Per-layer convolutional geometry: (text_seq_len, W, kernel) for a "conv" layer, where the image tokens form a
    W x W grid (image_seq_len = W^2), and None for any other layer."""
    kernel = validate_conv_kernel(kernel)
    if attention_types is None:
        return [None] * n_layers
    types = list(attention_types)
    if "conv" not in types:
        return [None] * len(types)
    W = math.isqrt(image_seq_len)
    if W * W != image_seq_len:
        raise ValueError(f"convolutional attention layers need a square image-token grid, but image_seq_len = "
                         f"{image_seq_len} is not a square")
    return [(int(text_seq_len), W, kernel) if t == "conv" else None for t in types]


SPARSE_BLOCK_SIZES = (16, 32, 64)


def _sparse_int(name, v, lo):
    if isinstance(v, bool) or not isinstance(v, numbers.Integral) or v < lo:
        raise ValueError(f"{name} must be an integer >= {lo}, got {v!r}")
    return int(v)


def validate_block_sparse(block_size, local_window_blocks, random_blocks, layout_seed, seq_len):
    """(block, window, random, seed) of block-sparse attention layers: sparse_block_size (16, the default, 32 or 64),
    sparse_local_window_blocks (an integer >= 1, default 4), sparse_random_blocks (an integer >= 0, default
    seq_len // block // 4, DALLE-pytorch's) and sparse_layout_seed (an integer >= 0, default 0).  None takes the
    default; anything else that is not such an integer raises a ValueError naming the key."""
    b = 16 if block_size is None else block_size
    if isinstance(b, bool) or not isinstance(b, numbers.Integral) or b not in SPARSE_BLOCK_SIZES:
        raise ValueError(f"sparse_block_size must be one of {SPARSE_BLOCK_SIZES}, got {block_size!r}")
    b = int(b)
    w = _sparse_int("sparse_local_window_blocks", 4 if local_window_blocks is None else local_window_blocks, 1)
    r = _sparse_int("sparse_random_blocks", seq_len // b // 4 if random_blocks is None else random_blocks, 0)
    seed = _sparse_int("sparse_layout_seed", 0 if layout_seed is None else layout_seed, 0)
    return b, w, r, seed


def block_sparse_layout(seq_len, text_seq_len, block, local_window_blocks, random_blocks, seed, owner):
    """The block layout of a block-sparse layer (DeepSpeed's VariableSparsityConfig as DALLE-pytorch configures it,
    unidirectional, one layout for every head): bool [nb, nb], nb = ceil(seq_len / block), where layout[r][c] lets the
    queries of block r see the keys of block c <= r.  An entry is set when
    - c < ceil(text_seq_len / block) (global blocks: the caption, vertical only);
    - c // w == r // w (local windows of w = local_window_blocks blocks aligned from block 0, the diagonal included);
    - c is one of min(R, r + 1) distinct blocks of [0, r] drawn at random, R = random_blocks: the rows r = 0 .. nb - 1
      in order, each rng.choice(r + 1, min(R, r + 1), replace=False) with rng = numpy.random.Generator(PCG64(
      SeedSequence([seed, owner]))).  owner is the layer that owns the token mixer (shared_attn_ids), so layers that
      share attention share the layout.
    The random draw is from the causal range [0, r], unlike DeepSpeed's (DESIGN.md).  A pure function of its
    arguments: the same on every rank and at generation time."""
    import numpy as np
    nb = -(-seq_len // block)
    lay = np.zeros((nb, nb), dtype=bool)
    rng = np.random.Generator(np.random.PCG64(np.random.SeedSequence([int(seed), int(owner)])))
    for r in range(nb):
        lay[r, rng.choice(r + 1, min(random_blocks, r + 1), replace=False)] = True
    idx = np.arange(nb)
    lay |= (idx[None, :] // local_window_blocks) == (idx[:, None] // local_window_blocks)
    lay[:, :-(-text_seq_len // block)] = True
    return np.tril(lay)


def layer_block_sparse(attention_types, text_seq_len, image_seq_len, n_layers, attn_owner=None, block_size=None,
                       local_window_blocks=None, random_blocks=None, layout_seed=None):
    """Per-layer block-sparse layout: block_sparse_layout of the layer's token-mixer owner for a "block_sparse" layer
    and None for any other.  The keys are validated (validate_block_sparse) whether or not such a layer exists."""
    S = text_seq_len + image_seq_len
    b, w, r, seed = validate_block_sparse(block_size, local_window_blocks, random_blocks, layout_seed, S)
    if attention_types is None:
        return [None] * n_layers
    owner = list(range(n_layers)) if attn_owner is None else attn_owner
    layouts = {o: block_sparse_layout(S, text_seq_len, b, w, r, seed, o)
               for o, t in zip(owner, attention_types) if t == "block_sparse"}
    return [layouts[owner[i]] if t == "block_sparse" else None for i, t in enumerate(attention_types)]


POSITION_EMBEDDINGS = ("absolute", "row_col")


def validate_position_embedding(value):
    """The image_position_embedding scheme: None or "absolute" (a learned vector per position, the reference's wpe) ->
    "absolute"; "row_col" (the DALL-E paper's row embedding + column embedding per image token); anything else is
    rejected."""
    if value is None:
        return "absolute"
    if not isinstance(value, str) or value not in POSITION_EMBEDDINGS:
        raise ValueError(f"image_position_embedding = {value!r}: must be one of {POSITION_EMBEDDINGS} (or null)")
    return value


def validate_per_position_padding(value):
    """per_position_padding: None or a bool (None: False)."""
    if value is None:
        return False
    if not isinstance(value, bool):
        raise ValueError(f"per_position_padding = {value!r}: must be true, false or null")
    return value


def validate_logits_mask(value):
    """logits_mask: None or a bool (None: False)."""
    if value is None:
        return False
    if not isinstance(value, bool):
        raise ValueError(f"logits_mask = {value!r}: must be true, false or null")
    return value


def image_grid_side(image_seq_len):
    """W of the W x W image-token grid row / column position embeddings need (image_seq_len = W^2)."""
    W = math.isqrt(image_seq_len)
    if W * W != image_seq_len:
        raise ValueError(f"row_col image position embeddings need a square image-token grid, but image_seq_len = "
                         f"{image_seq_len} is not a square")
    return W


def _real(v):
    return isinstance(v, numbers.Real) and not isinstance(v, bool)


def validate_loss_weights(text_loss_weight=None, image_loss_weight=None, z_loss=None):
    """((w_text, w_image) or None, z) of the weighted loss.  Both weights or neither, each a finite real >= 0 with a
    sum > 0; z a finite real >= 0 (None: 0)."""
    if (text_loss_weight is None) != (image_loss_weight is None):
        raise ValueError("text_loss_weight and image_loss_weight must be given together "
                         f"(got {text_loss_weight!r}, {image_loss_weight!r})")
    for name, v in (("text_loss_weight", text_loss_weight), ("image_loss_weight", image_loss_weight),
                    ("z_loss", z_loss)):
        if v is not None and not (_real(v) and math.isfinite(v) and v >= 0):
            raise ValueError(f"{name} = {v!r}: must be a finite real number >= 0")
    weights = None
    if text_loss_weight is not None:
        weights = (float(text_loss_weight), float(image_loss_weight))
        if weights[0] + weights[1] <= 0:
            raise ValueError("text_loss_weight + image_loss_weight must be > 0")
    return weights, 0.0 if z_loss is None else float(z_loss)


def loss_coefficients(loss_weights, text_seq_len, image_seq_len, global_batch):
    """(a_text, a_image): the coefficient of one text / image row's loss in the weighted loss
        (w_t sum_text l / (B (TL - 1)) + w_i sum_image l / (B (IL + 1))) / (w_t + w_i),  B = global_batch.
    A text row predicts a text token (positions p < TL - 1), an image row an image token or EOS.  Without weights
    (loss_weights None) every row carries 1 / (B S), the reference's mean over all positions."""
    n_text, n_image = text_seq_len - 1, image_seq_len + 1
    if loss_weights is None:
        a = 1.0 / (global_batch * (n_text + n_image))
        return a, a
    wt, wi = loss_weights
    a_text = wt / ((wt + wi) * global_batch * n_text) if n_text > 0 else 0.0
    return a_text, wi / ((wt + wi) * global_batch * n_image)


LAYERNORM_WIDTHS = (256, 512, 768, 1024, 2048, 4096)   # the d db200_layernorm_fwd / _bwd_ex dispatch (csrc/rowops.cu)
HEAD_DIMS = (64, 128)                                  # the head dims of the attention and decoding kernels


def _count(v):
    return isinstance(v, numbers.Integral) and not isinstance(v, bool)


def validate_geometry(n_embd, n_heads, text_seq_len, image_seq_len, text_vocab_size, image_vocab_size, n_layers=1):
    """The head dim n_embd // n_heads of a model the kernels can run, or an error naming the knob: ValueError for a
    malformed value, L.DB200Error for a width or head dim no kernel implements.

    n_embd must be one of LAYERNORM_WIDTHS and n_embd / n_heads one of HEAD_DIMS.  Every count must be an integer >= 1.
    text_seq_len >= 1 because the first image token is predicted at the last text position: without one, no row
    predicts it and generation has no position to draw it from.  text_vocab_size >= 1 because the caption padding id
    and the text window of the logits mask are text ids."""
    for name, v in (("n_embd", n_embd), ("n_heads", n_heads), ("n_layers", n_layers), ("text_seq_len", text_seq_len),
                    ("image_seq_len", image_seq_len), ("text_vocab_size", text_vocab_size),
                    ("image_vocab_size", image_vocab_size)):
        if not _count(v) or v < 1:
            raise ValueError(f"{name} must be an integer >= 1, got {v!r}")
    if n_embd % n_heads != 0:   # src/dalle_mtf/models.py:232
        raise ValueError(f"n_embd {n_embd} must be divisible by n_heads {n_heads}")
    if n_embd not in LAYERNORM_WIDTHS:
        raise L.DB200Error(f"n_embd {n_embd} unsupported by the LayerNorm kernels (one of {LAYERNORM_WIDTHS})")
    dh = n_embd // n_heads
    if dh not in HEAD_DIMS:
        raise L.DB200Error(f"head_dim {dh} = n_embd {n_embd} / n_heads {n_heads} unsupported by the attention kernels "
                           f"(one of {HEAD_DIMS})")
    return dh


ACTIVATIONS = ("relu", "gelu")


def validate_activation(activation):
    """The MLP nonlinearity: "relu" (the reference's default, mtf.relu) or "gelu" (mtf's tanh GELU); anything else
    (other spellings, booleans, numbers) is a ValueError."""
    if not isinstance(activation, str) or activation not in ACTIVATIONS:
        raise ValueError(f"activation must be one of {ACTIVATIONS}, got {activation!r}")
    return activation


def validate_gated_mlp(gated_mlp):
    """The gated MLP switch: a bool (numbers, strings and None are a ValueError here; the config key's null is
    handled by model_fns.gated_mlp)."""
    if not isinstance(gated_mlp, bool):
        raise ValueError(f"gated_mlp must be a bool, got {gated_mlp!r}")
    return gated_mlp


def validate_rotary(rotary_dim, rotary_base, head_dim):
    """(r, base) of rotary position embeddings, or None without them.  rotary_dim None: off (rotary_base must then be
    None too); otherwise an even integer 2 <= r <= head_dim.  rotary_base None is 10000, else a finite real > 1."""
    if rotary_dim is None:
        if rotary_base is not None:
            raise ValueError(f"rotary_base = {rotary_base!r} given without rotary_dim")
        return None
    if not _count(rotary_dim) or rotary_dim % 2 or not 2 <= rotary_dim <= head_dim:
        raise ValueError(f"rotary_dim = {rotary_dim!r}: must be an even integer with 2 <= rotary_dim <= head_dim "
                         f"{head_dim} (or null)")
    base = 10000.0 if rotary_base is None else rotary_base
    if not (_real(base) and math.isfinite(base) and base > 1):
        raise ValueError(f"rotary_base = {rotary_base!r}: must be a finite number > 1")
    return int(rotary_dim), float(base)


def validate_rotary_emb(rotary_emb, image_seq_len, rotary=None, image_position_embedding=None):
    """DALLE-pytorch's rotary embedding switch: None or False -> False; True -> True.  On, it needs a square image-token
    grid and excludes rotary_dim / rotary_base (the validated `rotary`, None when off) and any non-null
    image_position_embedding: the model then has no learned position embedding at all.  Anything else (1, "true", ...)
    is a ValueError."""
    if rotary_emb is None or rotary_emb is False:
        return False
    if rotary_emb is not True:
        raise ValueError(f"rotary_emb = {rotary_emb!r}: must be true, false or null")
    if math.isqrt(image_seq_len) ** 2 != image_seq_len:
        raise ValueError(f"rotary_emb needs a square image-token grid, but image_seq_len = {image_seq_len} is not a "
                         "square")
    if rotary is not None:
        raise ValueError("rotary_emb cannot be combined with rotary_dim / rotary_base (GPT-NeoX rotary embeddings)")
    if image_position_embedding is not None:
        raise ValueError(f"rotary_emb replaces the learned position embeddings: image_position_embedding must be null, "
                         f"got {image_position_embedding!r}")
    return True


def rotary_emb_freqs(dh, grid_w):
    """The ‡ constants of DALLE-pytorch's rotary embedding (DESIGN.md §4), in one place: (nf, theta, phi, y, t_image,
    t_text_axial) with rot = dh // 3 and nf = rot // 2 pairs per part; theta_j = 1 / 10000^(2j / rot) (rotary-
    embedding-torch's 'lang' frequencies of dim rot), phi_j = pi linspace(1, max_freq / 2, nf)[j] with max_freq 10
    (its 'pixel' frequencies), y = linspace(-1, 1, grid_w) the image-grid coordinate, t_image = 8192 the text-part
    position of every image token and t_text_axial = -10 the row / column coordinate of every text token.  All float32
    as torch computes them."""
    rot = dh // 3
    nf = rot // 2
    theta = 1.0 / (10000 ** (torch.arange(0, rot, 2)[:nf].float() / rot))
    phi = torch.linspace(1.0, 10 / 2, nf) * math.pi
    y = torch.linspace(-1.0, 1.0, grid_w)
    return nf, theta, phi, y, 8192.0, -10.0


def rotary_emb_table(text_len, grid_w, dh):
    """The fp32 [S, 2, 3 nf] table of the rope_emb kernels, S = text_len + grid_w^2 (rotary_emb_freqs): position p's
    3 nf cosines, then its sines.  Pair m < nf (part A) has the angle t theta_m with t = p for a text position and
    t_image for every image token; pair nf + j (part B) t phi_j with t = y[row] for an image token and t_text_axial for
    text; pair 2 nf + j (part C) the same with y[column].  The angle is the float32 product; its cos and sin are
    evaluated in float64 and rounded once to fp32."""
    nf, theta, phi, y, t_image, t_text_axial = rotary_emb_freqs(dh, grid_w)
    n_img = grid_w * grid_w
    t_a = torch.cat([torch.arange(text_len, dtype=torch.float32), torch.full((n_img,), t_image)])
    rows = y.repeat_interleave(grid_w)          # image token r W + c: row r
    cols = y.repeat(grid_w)                     # and column c
    t_b = torch.cat([torch.full((text_len,), t_text_axial), rows])
    t_c = torch.cat([torch.full((text_len,), t_text_axial), cols])
    angle = torch.cat([t_a[:, None] * theta[None, :], t_b[:, None] * phi[None, :], t_c[:, None] * phi[None, :]], 1)
    angle = angle.double()
    return torch.stack([torch.cos(angle), torch.sin(angle)], dim=1).to(F32)


def validate_sandwich_norm(sandwich_norm):
    """The sandwich LayerNorm switch: a bool (numbers, strings and None are a ValueError here; the config key's null is
    handled by model_fns.sandwich_norm)."""
    if not isinstance(sandwich_norm, bool):
        raise ValueError(f"sandwich_norm must be a bool, got {sandwich_norm!r}")
    return sandwich_norm


def validate_layer_scale(layer_scale):
    """The LayerScale setting: None or False -> None (off); True -> True (DALLE-pytorch's depth schedule,
    layer_scale_init); a finite real > 0 -> that float for every layer.  Anything else is a ValueError: in particular a
    bool is never read as the number 1 or 0."""
    if layer_scale is None or layer_scale is False:
        return None
    if layer_scale is True:
        return True
    if not (_real(layer_scale) and math.isfinite(layer_scale) and layer_scale > 0):
        raise ValueError(f"layer_scale = {layer_scale!r}: must be true, false, null or a finite number > 0")
    return float(layer_scale)


def layer_scale_init(layer_scale, i):
    """The initial value of layer i's (0-based) LayerScale vectors: a number as given, or for True DALLE-pytorch's
    schedule by depth n = i + 1: 0.1 for n <= 18, 1e-5 for 18 < n <= 24, 1e-6 beyond."""
    if layer_scale is not True:
        return float(layer_scale)
    n = i + 1
    return 0.1 if n <= 18 else 1e-5 if n <= 24 else 1e-6


STABLE_ALPHA = 0.1   # the stable option's embedding gradient shrink: tokens * 0.1 + tokens.detach() * 0.9


def validate_stable(stable):
    """The stable switch: None (off) or a bool; numbers, strings and other values are a ValueError."""
    if stable is None:
        return False
    if not isinstance(stable, bool):
        raise ValueError(f"stable must be a bool or None, got {stable!r}")
    return stable


def validate_share_input_output_emb(value):
    """share_input_output_emb: None or a bool (None: False); numbers, strings and other values are a ValueError."""
    if value is None:
        return False
    if not isinstance(value, bool):
        raise ValueError(f"share_input_output_emb must be a bool or None, got {value!r}")
    return value


def validate_shared_ids(ids, n_layers, name):
    """shared_attn_ids / shared_ff_ids (`name`): None (every layer its own module) or a non-empty list of integers >= 0,
    cycled to n_layers as DALLE-pytorch's cycle() does ([0, 1] at 6 layers: 0 1 0 1 0 1).  Returns the per-layer ids or
    None.  Bools, non-integers, negative ids, an empty list and anything but a list or tuple are a ValueError."""
    if ids is None:
        return None
    if not isinstance(ids, (list, tuple)) or not ids or any(not _count(v) or v < 0 for v in ids):
        raise ValueError(f"{name} = {ids!r}: must be null or a non-empty list of integers >= 0")
    return [int(ids[i % len(ids)]) for i in range(n_layers)]


def shared_owners(ids, n_layers):
    """Per layer, the owner of its shared module: the lowest layer with the same id (every layer its own without
    ids)."""
    if ids is None:
        return list(range(n_layers))
    first = {}
    return [first.setdefault(v, i) for i, v in enumerate(ids)]


def sharing_owners(shared_attn_ids, shared_ff_ids, n_layers, attention_types=None):
    """(attn_owner, ff_owner): per layer, the owner of its token mixer and of its MLP (shared_owners of the validated,
    cycled ids).  Layers that share an attention id must have the same attention type (DALLE-pytorch refuses it
    too): a ValueError names the first such pair."""
    attn_ids = validate_shared_ids(shared_attn_ids, n_layers, "shared_attn_ids")
    ff_ids = validate_shared_ids(shared_ff_ids, n_layers, "shared_ff_ids")
    attn_owner = shared_owners(attn_ids, n_layers)
    types = ["global"] * n_layers if attention_types is None else list(attention_types)
    for i, o in enumerate(attn_owner):
        if len(types) == n_layers and types[i] != types[o]:
            raise ValueError(f"shared_attn_ids: layers {o} and {i} share attention id {attn_ids[i]} but have different "
                             f"attention types ({types[o]!r}, {types[i]!r})")
    return attn_owner, shared_owners(ff_ids, n_layers)


def validate_shift_tokens(shift_tokens, image_seq_len):
    """The token-shift switch: a bool (numbers, strings and None are a ValueError here; the config key's null is
    handled by model_fns.shift_tokens).  On, it needs a square image-token grid (image_seq_len = W^2)."""
    if not isinstance(shift_tokens, bool):
        raise ValueError(f"shift_tokens must be a bool, got {shift_tokens!r}")
    if shift_tokens and math.isqrt(image_seq_len) ** 2 != image_seq_len:
        raise ValueError(f"shift_tokens needs a square image-token grid, but image_seq_len = {image_seq_len} is not "
                         f"a square")
    return shift_tokens


def rope_table(n_pos, rotary_dim, base):
    """The fp32 [n_pos, 2, rotary_dim / 2] table of the rotary kernels: position p's cos(p theta_j), then its
    sin(p theta_j), theta_j = base^(-2j / rotary_dim), each evaluated in float64 and rounded once to fp32."""
    h = rotary_dim // 2
    theta = torch.tensor([base ** (-2.0 * j / rotary_dim) for j in range(h)], dtype=torch.float64)
    angle = torch.arange(n_pos, dtype=torch.float64)[:, None] * theta[None, :]
    return torch.stack([torch.cos(angle), torch.sin(angle)], dim=1).to(F32)


class DalleEngine:
    """One data-parallel replica of the DALL-E decoder (src/dalle_mtf/models.py:141-416)."""

    VECTOR_PARAMS = ("ln1_g", "ln1_b", "o_b", "ln2_g", "ln2_b", "b1", "b2", "lna_g", "lna_b", "lnm_g", "lnm_b", "lnf_g",
                     "lnf_b", "bout", "gm_bin", "sgu_g", "sgu_b", "sgu_c", "gm_bout", "lsa", "lsm")
    conv = None   # per-layer conv geometry (layer_conv), set by the constructor; None: no conv layer
    block_sparse = None   # per-layer ops.BlockSparse (layer_block_sparse), set by the constructor; None: none
    gated_mlp = False   # the gated MLP (validate_gated_mlp), set by the constructor
    shift_tokens = False   # the token shift (validate_shift_tokens), set by the constructor
    sandwich_norm = False   # the sandwich LayerNorm (validate_sandwich_norm), set by the constructor
    mlp = ()   # per-layer flags of the gMLP token-mixing layers (layer_mlp), set by the constructor; () none
    layer_scale = None   # LayerScale (validate_layer_scale), set by the constructor; None: off
    stable = False   # DALLE-pytorch's stable option (validate_stable), set by the constructor
    tied = False   # share_input_output_emb (validate_share_input_output_emb), set by the constructor
    rotary_emb = False   # DALLE-pytorch's rotary embedding (validate_rotary_emb), set by the constructor

    def __init__(self, n_embd, n_layers, n_heads, text_vocab_size, image_vocab_size, text_seq_len, image_seq_len,
                 device="cuda", recompute_grad=False, attn_scale=1.0, ln_eps=1e-5, zero=None, dropout=(0.0, 0.0, 0.0),
                 dropout_seed=0, attention_types=None, local_attention_radius=256, loss_weights=None, z_loss=0.0,
                 conv_attention_kernel=5, image_position_embedding=None, per_position_padding=False,
                 activation="relu", logits_mask=False, rotary_dim=None, rotary_base=None, gated_mlp=False,
                 shift_tokens=False, sandwich_norm=False, layer_scale=None, stable=False, share_input_output_emb=False,
                 shared_attn_ids=None, shared_ff_ids=None, sparse_block_size=16, sparse_local_window_blocks=4,
                 sparse_random_blocks=None, sparse_layout_seed=0, rotary_emb=None):
        """dropout = (embed_dropout, attention_dropout, residual_dropout) rates in [0, 1) (src/dalle_mtf/models.py:
        198-200, 215-217, 290-299, 312-314, 321-323).  They apply only to a forward() given a `step`; the masks are a
        pure function of (dropout_seed, step, site, global element index) (include/dalle_b200.h, D0).

        attention_types: one "global", "local", "axial_row", "axial_col" or "conv" per layer (None: every layer
        global).  A local layer attends from position i to positions (i - local_attention_radius, i]
        (src/dalle_mtf/models.py:257-273).  Axial and conv layers need image_seq_len = W^2: text positions attend
        causally, and the image token at grid row r, column c attends to every text position and to the image tokens
        of row r at columns <= c (axial_row), of column c at rows <= r (axial_col), or at rows (r - k, r] and columns
        (c - k, c] with k = conv_attention_kernel (conv, DALL-E's convolutional mask).  Local, axial and conv layers
        apply no attention dropout (the reference passes local attention none, :270; the dropout site 2 + 3l of such a
        layer l is unused); their residual dropout is unchanged.

        zero: a DataParallel with world > 1 turns on optimiser-state sharding (ZeRO-1, SURVEY.md §7 "12 B in pure
        DP"): fp32 master / Adam m / Adam v exist only for this rank's 1/N slice of the flat buffer, the bf16 compute
        copy and the fp32 gradients stay full; after the (all-reduced) gradients are final every rank updates its
        slice and the bf16 parameters are all-gathered in place.  Still data parallel: same batch split, same maths.

        loss_weights = (w_text, w_image) and z_loss: the weighted loss of loss_coefficients() with z_loss * lse^2 added
        to every row (validate_loss_weights).  With either active, forward() accumulates four sums (weighted loss,
        text-row CE, image-row CE, z-term) and backward() runs the weighted CE_GRAD epilogue; otherwise the step is
        the reference's.

        image_position_embedding "row_col" (None / "absolute": the reference's wpe [S, d]): wpe holds the text
        positions only and image token (r, c) of the W x W grid (image_seq_len = W^2) gets image_row[r] + image_col[c].
        The engine composes one bf16 [S, d] table from the bf16 parameters (pos_table) wherever they are rewritten, and
        every embedding kernel reads it as it reads wpe otherwise; backward folds the table's gradient into the three.

        per_position_padding: the text vocabulary grows by text_seq_len padding tokens, token text_vocab_size + p
        being text position p's pad (pad_base = text_vocab_size), and image code i becomes token image_offset + i with
        image_offset = text_vocab_size + text_seq_len (otherwise text_vocab_size).  Captions are mapped by
        ops.assemble_tokens_pp.

        activation: the MLP nonlinearity (validate_activation).  "gelu" makes the MLP gelu(LN2(x) W1 + b1) W2 + b2 with
        mtf's tanh GELU, fused into the W1 product's epilogue (which also keeps the pre-activation z for backward: one
        more bf16 [T, 4d] per saved layer) and into its dgrad's; no parameter changes.

        logits_mask (DALLE-pytorch's logits_mask): a text row (position p < text_seq_len - 1, whose target is a text
        token) normalises over the ids [0, image_offset), an image row (target an image code or EOS) over
        [image_offset, V); each row's loss is lse_window - logit[label] (+ z_loss lse_window^2) and its gradient is 0
        outside the window.  The step gathers each class into one block of rows and runs the vocabulary products on
        that block's columns only (_masked_forward / _masked_backward); logits() returns -inf outside the windows.  A
        label outside its row's window is undefined, as a label >= V is: assemble_tokens(_pp) keeps every label in its
        window as long as the caption ids are < text_vocab_size and the codes < image_vocab_size.  No parameter
        changes; prefill and decoding are unchanged (image draws already see only image ids).

        rotary_dim r (None: off) and rotary_base (None: 10000): rotary position embeddings, GPT-NeoX's rotate_half
        layout with partial rotary (validate_rotary).  After the q|k|v product, the pair (x_j, x_{j+r/2}) of the first r
        dims of every q and k head of every layer is rotated by p theta_j, p the token's sequence index and theta_j =
        base^(-2j/r), in fp32 and rounded to bf16 (ops.rope_fwd); backward applies the transpose to dq and dk, and the
        decoder rotates each step's q and k before they reach the cache.  v, the attention scale and the learned
        position embeddings are unchanged, and no parameter is added.

        gated_mlp (validate_gated_mlp): the MLP becomes DALLE-pytorch's gated FeedForward, y = LN2(x) W1 + b1 with W1
        [d, 8d], zv, zg = bf16(y[:, :4d]), bf16(y[:, 4d:]), h = bf16(zv bf16(act(zg))), out = h W2 + b2, with act the
        `activation` (ReGLU or GEGLU).  The gate is fused into the W1 product's epilogue, which keeps z = [zv | zg]
        ([T, 8d] bf16 per saved layer) for backward, and into its dgrad's.

        shift_tokens (validate_shift_tokens): DALLE-pytorch's token shift after both LayerNorms of every layer (its
        PreNorm(PreShiftToken(...))).  With c = d / 4, a text position's columns [0, 2c) come from the position before
        it, an image token's [0, c) from the token one grid row above and [c, 2c) from the token to its left, zeros
        where there is none; [2c, d) are kept (ops.shift_tokens_fwd, exact copies).  The LayerNorm writes a scratch
        [T, d] and the shift writes the ln1 / ln2 buffers the q|k|v and W1 products and their wgrads read; backward
        applies the transpose to d(LN out) before the LayerNorm backward, and the decoder keeps a [rows, S, d/2] cache
        of unshifted outputs per layer and LayerNorm.  No parameter is added.

        sandwich_norm (validate_sandwich_norm): CogView's Sandwich-LN as DALLE-pytorch's PreNorm(..., sandwich=True)
        builds it.  Each branch output after its residual dropout, oa = drop(a Wo + o_b) and om = drop(h W2 + b2), is
        normalised by its own LayerNorm before the residual add: xmid = x + LNa(oa), xout = xmid + LNm(om), one
        rounding each (ops.layernorm_residual_fwd); LNa / LNm are the parameters lna_g / lna_b and lnm_g / lnm_b
        (layer_i/attn/norm_out and layer_i/mlp/norm_out), g = 1 and b = 0 at initialisation, not weight-decayed.  oa,
        om and their statistics are kept per saved layer (two bf16 [T, d] and four fp32 [T]).

        An "mlp" entry of attention_types makes that layer a gMLP block (DALLE-pytorch's gMLPBlock with dim_ff = 4d,
        causal, one head) in place of attention: u = gelu(LN1(x) W_in + b_in) (bf16, mtf's tanh GELU; the GELU
        epilogue keeps z), res, gate = u[:, :2d], u[:, 2d:], gn = bf16(LN_sgu(gate)), mixed_i = sum_{j <= i} W_sgu[i, j]
        gn_j + c_sgu[i] in fp32 per sequence, h = bf16(mixed res), and x += drop(h W_out + b_out) (with the sandwich
        LayerNorm, LNa of it).  W_sgu [S, S] is lower triangular: its strict upper triangle starts, and stays, exactly
        0 (its gradient there is never written) and a checkpoint with a non-zero one is refused.  Rotary embeddings and
        attention dropout do not apply to the layer; residual dropout does.  Kept per saved layer: res, gate, their z,
        gn, mixed and h (seven bf16 [T, 2d]) and the SGU LayerNorm's statistics.

        layer_scale (validate_layer_scale): DALLE-pytorch's LayerScale around both branches of every layer.  The branch
        output after its residual dropout (with the sandwich LayerNorm: that LayerNorm's output) is multiplied per
        channel by a learned vector before the residual add, xmid = bf16(x + s_a oa), xout = bf16(xmid + s_m om), one
        rounding each in fp32 (ops.layer_scale_residual_fwd, ops.layernorm_scale_residual_fwd).  s_a and s_m are the
        parameters lsa and lsm (layer_i/attn/layer_scale, or layer_i/gmlp/layer_scale in a gMLP layer, and
        layer_i/mlp/layer_scale), initialised by layer_scale_init and not weight-decayed.  Without the sandwich
        LayerNorm oa and om are kept per saved layer (two bf16 [T, d]); with it they are already kept.

        stable (validate_stable): DALLE-pytorch's stable option.  (1) The embedding's gradient shrinks: its forward is
        unchanged and every embedding table's gradient is STABLE_ALPHA times what it was (tokens * alpha +
        tokens.detach() * (1 - alpha)).  (2) DivideMax before the final LayerNorm, wherever it runs (training, the
        prefill, the decoder, logits()): per row m = max_c x[c] (held constant in backward), u = x / m in fp32 and
        hf = bf16(LN_f(u)) (ops.layernorm_divmax_fwd); one more fp32 [T] keeps m.  (3) Its stable softmax is the
        softmax every attention kernel already computes (the row maximum subtracted in fp32).  No parameter is
        added.

        share_input_output_emb (validate_share_input_output_emb): DALLE-pytorch's tied embedding.  wte [Vpad, d] is
        both the input embedding and the vocabulary projection, logits = hf wte^T + bout; wout does not exist
        (to_logits/linear_out/kernel is not a variable), bout stays and so does the EOS row of wte.  The vocabulary
        products read wte as a K-major B operand; wte's gradient is the sum of the vocabulary wgrad and the embedding
        gather's (which alone `stable` shrinks).  wte's pad rows V..Vpad-1 start and stay exactly 0.

        shared_attn_ids / shared_ff_ids (validate_shared_ids): DALLE-pytorch's parameter sharing.  Layers with the same
        (cycled) attention id use one token mixer (wqkv, wo, o_b, or a gMLP layer's GMLP_MODULE), layers with the same
        ff id one MLP (w1, b1, w2, b2).  LayerNorms, sandwich LayerNorms, LayerScale and decode caches stay per layer.
        A shared module belongs to its lowest user (attn_owner / ff_owner): it is initialised and checkpointed there,
        and the other users' names are layout aliases of its entries, so their gradients add into its slot.  Layers
        sharing an attention id must have the same attention type.

        A "block_sparse" entry of attention_types makes that layer DeepSpeed-style block-sparse attention
        (DALLE-pytorch's SparseAttention): query i sees key j <= i iff layout[i // b][j // b] of block_sparse_layout,
        with b = sparse_block_size, the local window sparse_local_window_blocks, sparse_random_blocks random blocks per
        row and sparse_layout_seed (validate_block_sparse).  The layout is drawn per token-mixer owner and is the same
        for every head; it is not a variable, so sampling must use the training config's keys.  No attention dropout
        (the layer's site is unused); residual dropout is unchanged.

        rotary_emb (validate_rotary_emb): DALLE-pytorch's rotary embedding in place of learned positions.  After the
        q|k|v product, the interleaved pairs (2m, 2m+1), m < 3 nf, of every q, k and v head of every attention layer
        are rotated by the angles of rotary_emb_table (text position, image row, image column; gMLP layers are not
        rotated), in fp32 and rounded to bf16 (ops.rope_emb_fwd); backward applies the transpose to d(q|k|v), and the
        decoder rotates each step's q, k and v before k and v reach the cache.  There is no wpe: the embedding kernels
        read an all-zero bf16 [S, d] table the engine owns (pos_table), and their position gradient goes to a scratch
        nothing reads (_dpos)."""
        self.dh = validate_geometry(n_embd, n_heads, text_seq_len, image_seq_len, text_vocab_size, image_vocab_size,
                                    n_layers)
        self.shift_tokens = validate_shift_tokens(shift_tokens, image_seq_len)
        self.shift_w = math.isqrt(image_seq_len) if self.shift_tokens else None   # the grid side W
        self.sandwich_norm = validate_sandwich_norm(sandwich_norm)
        self.layer_scale = validate_layer_scale(layer_scale)
        self.stable = validate_stable(stable)
        self.rotary = validate_rotary(rotary_dim, rotary_base, self.dh)
        self.rotary_emb = validate_rotary_emb(rotary_emb, image_seq_len, self.rotary, image_position_embedding)
        self.activation = validate_activation(activation)
        self.gated_mlp = validate_gated_mlp(gated_mlp)
        self.glu = self.activation if self.gated_mlp else None   # the gate's nonlinearity, or None: no gate
        self.gelu = self.activation == "gelu" and not self.gated_mlp    # the ungated GELU MLP
        # linear_fwd keywords of an inference W1
        self.mlp_act = {"glu": self.glu} if self.gated_mlp else {"gelu": True} if self.gelu else {"relu": True}
        self.row_col = validate_position_embedding(image_position_embedding) == "row_col"
        self.grid_w = image_grid_side(image_seq_len) if self.row_col else None
        self.per_position_padding = validate_per_position_padding(per_position_padding)
        self.tied = validate_share_input_output_emb(share_input_output_emb)
        self.attn_owner, self.ff_owner = sharing_owners(shared_attn_ids, shared_ff_ids, n_layers, attention_types)
        L.require_device()
        self.d, self.L, self.H = n_embd, n_layers, n_heads
        self.text_vocab_size, self.image_vocab_size = text_vocab_size, image_vocab_size
        self.text_seq_len, self.image_seq_len = text_seq_len, image_seq_len
        self.S = text_seq_len + image_seq_len                       # models.py:153
        self.pad_base = text_vocab_size if self.per_position_padding else None
        self.image_offset = text_vocab_size + (text_seq_len if self.per_position_padding else 0)
        self.V = self.image_offset + image_vocab_size + 1           # models.py:157 (extra id = EOS)
        self.eos_token_id = self.V - 1                              # models.py:158
        self.Vpad = _round_up(self.V, 64)
        self.logits_mask = validate_logits_mask(logits_mask)
        # windows of the masked vocabulary products: the text block over columns [0, mask_text_cols) (n_valid =
        # image_offset), the image block over [mask_c0, mask_c0 + mask_image_cols) (n_valid = V - mask_c0), with
        # mask_c0 = image_offset rounded down to 8 columns so that the operand base stays 16-byte aligned for TMA
        self.text_rows = text_seq_len - 1
        self.mask_c0 = self.image_offset // 8 * 8
        self.mask_text_cols = _round_up(self.image_offset, 8)
        self.mask_image_cols = _round_up(self.V - self.mask_c0, 8)
        self.device = torch.device(device)
        self.recompute_grad = bool(recompute_grad)
        self.attn_scale = float(attn_scale)
        self.ln_eps = float(ln_eps)
        self.dropout = tuple(float(r) for r in dropout)
        if len(self.dropout) != 3:
            raise ValueError("dropout = (embed, attention, residual) rates")
        for r in self.dropout:
            L.dropout_threshold(r)   # rejects a rate outside [0, 1)
        self.dropout_seed = int(dropout_seed)
        self._drop = None            # descriptors of the current forward (None: no dropout)
        # per layer: None (global, causal attention) or the window radius of a local layer
        self.radii = layer_radii(attention_types, local_attention_radius, n_layers)
        # per layer: None or the (text_len, grid_w, axis) of an axial layer, and the attention ops' keyword for it
        self.axial = layer_axial(attention_types, text_seq_len, image_seq_len, n_layers)
        self.axial_kw = [{} if a is None else {"axial": a} for a in self.axial]
        # per layer: None or the (text_len, grid_w, kernel) of a conv layer, and the attention ops' keyword for it
        self.conv = layer_conv(attention_types, text_seq_len, image_seq_len, conv_attention_kernel, n_layers)
        self.conv_kw = [{} if c is None else {"conv": c} for c in self.conv]
        # per layer: None or the ops.BlockSparse of a block-sparse layer (one per token-mixer owner), and its keyword
        sparse = validate_block_sparse(sparse_block_size, sparse_local_window_blocks, sparse_random_blocks,
                                       sparse_layout_seed, self.S)
        layouts = layer_block_sparse(attention_types, text_seq_len, image_seq_len, n_layers, self.attn_owner,
                                     *sparse)
        tables = {id(lay): ops.BlockSparse(lay, sparse[0], self.S, self.device) for lay in layouts if lay is not None}
        self.block_sparse = [None if lay is None else tables[id(lay)] for lay in layouts]
        self.block_sparse_kw = [{} if m is None else {"block_sparse": m} for m in self.block_sparse]
        # per layer: True for a gMLP token-mixing layer
        self.mlp = layer_mlp(attention_types, n_layers, self.S, n_embd)
        lw = (None, None) if loss_weights is None else tuple(loss_weights)
        self.loss_weights, self.z_loss = validate_loss_weights(*lw, z_loss)
        self.weighted_loss = self.loss_weights is not None or self.z_loss > 0
        self._cew = None             # lib.CeWeights of the current forward (weighted loss only; logits mask: a
                                     # (text block, image block) pair)

        d, V, S, Lyr = self.d, self.V, self.S, self.L
        mlp_layers = self.mlp if any(self.mlp) else None
        kw = dict(gated_mlp=self.gated_mlp, sandwich_norm=self.sandwich_norm, mlp_layers=mlp_layers,
                  layer_scale=self.layer_scale is not None, tied=self.tied, attn_owner=self.attn_owner,
                  ff_owner=self.ff_owner, wpe=not self.rotary_emb)
        self.layout = lay = param_layout(d, Lyr, V, S, text_seq_len, self.grid_w, **kw) if self.row_col else \
            param_layout(d, Lyr, V, S, **kw)
        self.embed_names = ("wte", "wpe", "image_row", "image_col") if self.row_col else \
            ("wte",) if self.rotary_emb else ("wte", "wpe")
        self.n_params_padded = lay.size
        # trailing 64 floats of the gradient buffer carry scalars that ride along with the gradient all-reduce:
        #   [0] = sum of per-token losses of this rank (weighted loss: sum of a_t * loss_t)
        #   [1..3] = weighted loss only: text-row CE sum, image-row CE sum, z-term sum
        self.aux_off = lay.size
        n = lay.size + 64
        dev = self.device
        self._views = {}
        self.zero = zero if (zero is not None and getattr(zero, "world", 1) > 1) else None
        self.grads = torch.zeros(n, dtype=F32, device=dev)
        if self.zero is None:
            self.master = torch.zeros(n, dtype=F32, device=dev)
            self.adam_m = torch.zeros(n, dtype=F32, device=dev)
            self.adam_v = torch.zeros(n, dtype=F32, device=dev)
            self.shadow = torch.zeros(n, dtype=BF16, device=dev)
            self.shard = (0, lay.size)
        else:
            w, r = self.zero.world, self.zero.rank
            self.chunk = _round_up(-(-lay.size // w), 64)                 # elements per rank (equal: in-place all-gather)
            self.shard = (min(r * self.chunk, lay.size), min((r + 1) * self.chunk, lay.size))
            self.master = torch.zeros(self.chunk, dtype=F32, device=dev)  # this rank's slice only
            self.adam_m = torch.zeros(self.chunk, dtype=F32, device=dev)
            self.adam_v = torch.zeros(self.chunk, dtype=F32, device=dev)
            self.shadow = torch.zeros(max(w * self.chunk, n), dtype=BF16, device=dev)
            # compact fp32 copy of the vector parameters (LayerNorm g / b, biases) the kernels read in fp32: rebuilt
            # from the bf16 parameters after every all-gather — mtf casts every variable to the activation dtype when
            # it is used (src/dalle_mtf/ops.py:76-82), so this is the reference's own bf16 policy
            self._vec_off, table, off = {}, [], 0
            for name in lay.order:
                if name.split(".")[-1] in self.VECTOR_PARAMS:
                    o, shp = lay.entries[name]
                    self._vec_off[name] = (off, shp)
                    table += [o, off, shp[0]]
                    off += _round_up(shp[0], 64)
            for name, owner in lay.aliases.items():   # a shared vector reads its owner's slot
                if owner in self._vec_off:
                    self._vec_off[name] = self._vec_off[owner]
            self.vec32 = torch.zeros(off, dtype=F32, device=dev)
            self._vec_table = torch.tensor(table, dtype=torch.int64, device=dev)
        # the composed bf16 position table the embedding kernels read, and its fp32 gradient (rotary_emb: all zeros,
        # and a scratch gradient nothing reads)
        if self.row_col or self.rotary_emb:
            self.pos_table = torch.zeros(S, d, dtype=BF16, device=dev)
            self._dpos = torch.zeros(S, d, dtype=F32, device=dev)
        self.gnorm_sq = torch.zeros(1, dtype=F32, device=dev)
        # rotary position embeddings: r (None: off) and the cos / sin table of every position, built once
        self.rotary_dim = self.rotary[0] if self.rotary else None
        self.rope_table = rope_table(S, *self.rotary).to(dev) if self.rotary else None
        # rotary_emb: the cos / sin table of the text, row and column angles of every position, built once
        self.rope_emb_table = rotary_emb_table(text_seq_len, math.isqrt(image_seq_len), self.dh).to(dev) \
            if self.rotary_emb else None
        self._grads_clean = False
        self._bufs = None
        self._buf_key = None

    # ------------------------------------------------------------------------------------------ parameters
    # The flat buffers are allocated once and only ever written in place, so the per-name views are cached: building a
    # slice + view costs a few microseconds of host time, and the decode loop asks for ~70 of them per position.
    def _view(self, which, flat, name):
        key = (which, name)
        v = self._views.get(key)
        if v is None:
            v = self._views[key] = self.layout.view(flat, name)
        return v

    def P(self, name):  # fp32 view of a parameter (ZeRO-1: only the vector parameters exist in full fp32)
        if self.zero is not None:
            if name not in self._vec_off:
                raise L.DB200Error(f"{name}: the fp32 master of a matrix is sharded across ranks in ZeRO-1 mode")
            key = (3, name)
            v = self._views.get(key)
            if v is None:
                off, shp = self._vec_off[name]
                v = self._views[key] = self.vec32[off:off + shp[0]]
            return v
        return self._view(0, self.master, name)

    def W(self, name):  # bf16 compute copy
        return self._view(1, self.shadow, name)

    def G(self, name):  # fp32 gradient view
        return self._view(2, self.grads, name)

    def wte_rows(self, flat):
        """The [V, d] embedding rows of wte in the flat buffer `flat` (a tied wte has Vpad rows, the last ones pad)."""
        v = self.layout.view(flat, "wte")
        return v[:self.V] if self.tied else v

    def embed_table(self):
        """The bf16 [V, d] table the embedding kernels gather from."""
        return self.W("wte")[:self.V] if self.tied else self.W("wte")

    # The vocabulary products over the columns [c0, c0 + n) of the logits (default: all Vpad).  Untied, the B operand
    # is wout's [d, n] column window, MN-major; tied, it is wte's [n, d] row window, K-major (ldb = d).
    def _vocab_b(self, c0, n):
        if self.tied:
            w = self.W("wte")
            return (w if n is None else w[c0:c0 + n]), False
        w = self.W("wout")
        return (w if n is None else w[:, c0:c0 + n]), True

    def vocab_gemm(self, hf, out, c0=0, n=None, **kw):
        """logits (or a vocabulary epilogue over them) of the rows hf [M, d] against the columns [c0, c0 + n)."""
        b, b_mn = self._vocab_b(c0, n)
        return ops.gemm(hf, b, out, hf.shape[0], self.Vpad if n is None else n, self.d, a_mn=False, b_mn=b_mn, **kw)

    def vocab_wgrad(self, hf, dlogits, c0=0, n=None):
        """The vocabulary weight's gradient += from dlogits [M, n]: G(wout)[:, window] += hf^T dlogits, or tied
        G(wte)[window] += dlogits^T hf (the same both-MN-major product with M and N swapped)."""
        if self.tied:
            g = self.G("wte")
            return ops.linear_wgrad(dlogits, hf, g if n is None else g[c0:c0 + n])
        g = self.G("wout")
        return ops.linear_wgrad(hf, dlogits, g if n is None else g[:, c0:c0 + n])

    def vocab_dgrad(self, dlogits, out, c0=0, n=None):
        """out [M, d] = dlogits [M, n] times the vocabulary weight's window transposed (tied: wte[window], MN-major)."""
        b, b_mn = self._vocab_b(c0, n)
        if self.tied:
            return ops.linear_fwd(dlogits, b, out)
        return ops.linear_dgrad(dlogits, b, out)

    def pos_embedding(self):
        """The bf16 [S, d] position table the embedding kernels read: wpe, or with row / column image positions the
        table composed from wpe, image_row and image_col; with rotary_emb an all-zero table."""
        return self.pos_table if self.row_col or self.rotary_emb else self.W("wpe")

    def _compose_pos(self):
        """Rebuild the composed position table from the bf16 parameters (row / column image positions only)."""
        if self.row_col:
            ops.pos_compose(self.W("wpe"), self.W("image_row"), self.W("image_col"), self.pos_table)

    def n_params(self):
        """Trainable parameter count as the reference would print it (src/utils/utils.py:55-70)."""
        d, V, S, Lyr = self.d, self.V, self.S, self.L
        n_pos = (self.text_seq_len + 2 * self.grid_w) if self.row_col else 0 if self.rotary_emb else S
        gate = (4 * d * d + 4 * d) if self.gated_mlp else 0   # the gate half of W1 and b1
        sandwich = 4 * d if self.sandwich_norm else 0         # LNa and LNm: g and b each
        scales = 2 * d if self.layer_scale is not None else 0  # the two LayerScale vectors
        n_mlp = sum(self.mlp)
        # a gMLP layer: W_in + b_in, the SGU norm, W_sgu + c_sgu and W_out + b_out in place of q, k, v, o and o_b
        gmlp = 4 * d * d + 4 * d + 4 * d + S * S + S + 2 * d * d + d - (4 * d * d + d)
        n = V * d + n_pos * d + Lyr * (2 * d + 3 * d * d + d * d + d + 2 * d + 4 * d * d + 4 * d + 4 * d * d + d +
                                       gate + sandwich + scales) + n_mlp * gmlp + 2 * d + d * V + V
        if self.tied:   # no wout
            n -= d * V
        w1_cols = 8 * d if self.gated_mlp else 4 * d
        for i in range(Lyr):   # a shared module counts once, at its owner
            if not self._owns_mixer(i):
                n -= gmlp + 4 * d * d + d if self._is_mlp(i) else 4 * d * d + d
            if not self._owns_ff(i):
                n -= d * w1_cols + w1_cols + 4 * d * d + d
        return n

    EMBED_REF_NAMES = {"wte": "embedding/wte", "wpe": "positional_embedding/wpe",
                       "image_row": "positional_embedding/image_row", "image_col": "positional_embedding/image_col"}

    def _ref_embed_name(self, name):
        """Reference-style variable name of an embedding parameter (other names are returned unchanged)."""
        return self.EMBED_REF_NAMES.get(name, name)

    GMLP_REF_NAMES = {"gm_win": "gmlp/proj_in/kernel", "gm_bin": "gmlp/proj_in/bias", "sgu_g": "gmlp/sgu/norm/g",
                      "sgu_b": "gmlp/sgu/norm/b", "sgu_w": "gmlp/sgu/weight", "sgu_c": "gmlp/sgu/bias",
                      "gm_wout": "gmlp/proj_out/kernel", "gm_bout": "gmlp/proj_out/bias"}

    @staticmethod
    def _ref_names(i, sandwich_norm=False, mlp=False, layer_scale=False):
        pre = f"layer_{i}/"
        names = {
            "ln1_g": pre + "norm_1/g", "ln1_b": pre + "norm_1/b", "wo": pre + "attn/o",
            "o_b": pre + "attn/compute_output_bias/o_b", "ln2_g": pre + "norm_2/g", "ln2_b": pre + "norm_2/b",
            "w1": pre + "mlp/mlp_linear_1/kernel", "b1": pre + "mlp/mlp_linear_1/bias",
            "w2": pre + "mlp/mlp_linear_2/kernel", "b2": pre + "mlp/mlp_linear_2/bias",
        }
        if mlp:   # a gMLP layer: its token-mixing variables replace attn/o and o_b (and q, k, v)
            del names["wo"], names["o_b"]
            names.update({k: pre + v for k, v in DalleEngine.GMLP_REF_NAMES.items()})
        if sandwich_norm:
            names.update({"lna_g": pre + "attn/norm_out/g", "lna_b": pre + "attn/norm_out/b",
                          "lnm_g": pre + "mlp/norm_out/g", "lnm_b": pre + "mlp/norm_out/b"})
        if layer_scale:
            names.update({"lsa": pre + ("gmlp" if mlp else "attn") + "/layer_scale", "lsm": pre + "mlp/layer_scale"})
        return names

    @property
    def split_branch(self):
        """Whether each branch output is stored before its residual add (sandwich LayerNorm or LayerScale), its
        gradient then coming from the branch's own backward rather than from the LayerNorm that forms the residual
        gradient."""
        return self.sandwich_norm or self.layer_scale is not None

    def layer_last(self, i):
        """The last entry layer i owns in the layout: the end of its data-parallel bucket (a shared MLP's b2 belongs to
        its owner's bucket)."""
        p = f"l{i}."
        return p + ("lsm" if self.layer_scale is not None else "lnm_b" if self.sandwich_norm else
                    "b2" if self._owns_ff(i) else "ln2_b")

    def _is_mlp(self, i):
        """Whether layer i is a gMLP token-mixing layer."""
        return bool(self.mlp) and self.mlp[i]

    attn_owner = ff_owner = None   # per layer, the owner of its token mixer / MLP (sharing_owners); None: itself

    def _owns_mixer(self, i):
        """Whether layer i owns its token mixer (no shared_attn_ids, or the lowest layer of its id)."""
        return self.attn_owner is None or self.attn_owner[i] == i

    def _owns_ff(self, i):
        """Whether layer i owns its MLP (no shared_ff_ids, or the lowest layer of its id)."""
        return self.ff_owner is None or self.ff_owner[i] == i

    def _layer_ref_names(self, i):
        """Reference names of layer i's parameters other than q / k / v (with this engine's sandwich_norm, layer kind
        and layer_scale), without those of a shared module layer i does not own."""
        names = self._ref_names(i, self.sandwich_norm, self._is_mlp(i), self.layer_scale is not None)
        drop = (() if self._owns_mixer(i) else ATTN_MODULE + GMLP_MODULE) + (() if self._owns_ff(i) else FF_MODULE)
        return {k: v for k, v in names.items() if k not in drop}

    def _module_ref_names(self, i):
        """[(owner, what, reference names)] of layer i's token mixer and MLP, whatever layer owns them."""
        pre = f"layer_{i}/"
        ref = self._ref_names(i, mlp=self._is_mlp(i))
        mixer = [ref[k] for k in GMLP_MODULE] if self._is_mlp(i) else \
            [pre + "attn/q", pre + "attn/k", pre + "attn/v", ref["wo"], ref["o_b"]]
        return [(self.attn_owner[i] if self.attn_owner else i, "token mixer (shared_attn_ids)", mixer),
                (self.ff_owner[i] if self.ff_owner else i, "MLP (shared_ff_ids)", [ref[k] for k in FF_MODULE])]

    OUT_KERNEL = "to_logits/linear_out/kernel"

    def _check_sharing_names(self, named):
        """Refuse a checkpoint of another tying or sharing kind: an output projection kernel in the checkpoint of a
        tied model or none in an untied one's, a variable of a module the layer does not own, a missing one of a
        module it owns.  The error names the first such variable (layer order, the token mixer's first)."""
        if self.tied and self.OUT_KERNEL in named:
            raise L.DB200Error(f"load_params: {self.OUT_KERNEL}: an output projection, but this model ties it to "
                               "embedding/wte (share_input_output_emb)")
        if not self.tied and self.OUT_KERNEL not in named:
            raise L.DB200Error(f"load_params: {self.OUT_KERNEL}: missing from the checkpoint of a model without "
                               "share_input_output_emb")
        for i in range(self.L):
            for owner, what, names in self._module_ref_names(i):
                for rn in names:
                    if owner == i and rn not in named:
                        raise L.DB200Error(f"load_params: {rn}: missing from the checkpoint, and layer {i} owns its "
                                           f"{what}")
                    if owner != i and rn in named:
                        raise L.DB200Error(f"load_params: {rn}: layer {i} uses the {what} of layer {owner} and has "
                                           "no variable of its own")

    def _check_layer_kinds(self, named):
        """Refuse a checkpoint whose layer kinds differ from this model's: an attention layer's variables where this
        model has a gMLP layer, or the reverse; and a gMLP mixing weight whose strict upper triangle is not zero (the
        layer's causality).  The error names the first such variable."""
        for i in range(self.L):
            pre = f"layer_{i}/"
            if self._is_mlp(i):
                for rn in [pre + "attn/q", pre + "attn/k", pre + "attn/v", pre + "attn/o"]:
                    if rn in named:
                        raise L.DB200Error(f"load_params: {rn}: an attention variable, but layer {i} of this model is "
                                           "a gMLP ('mlp') layer")
                if not self._owns_mixer(i):   # its gMLP variables are its owner's (_check_sharing_names)
                    continue
                for v in self.GMLP_REF_NAMES.values():
                    if pre + v not in named:
                        raise L.DB200Error(f"load_params: {pre + v}: missing from the checkpoint of a model whose layer "
                                           f"{i} is a gMLP ('mlp') layer")
                w = named[pre + "gmlp/sgu/weight"]
                if tuple(w.shape) == (self.S, self.S) and bool(torch.triu(w, diagonal=1).ne(0).any()):
                    raise L.DB200Error(f"load_params: {pre}gmlp/sgu/weight: the strict upper triangle of the causal "
                                       "mixing weight must be exactly 0")
            else:
                extra = sorted(k for k in named if k.startswith(pre + "gmlp/"))
                if extra:
                    raise L.DB200Error(f"load_params: {extra[0]}: a gMLP variable, but layer {i} of this model is an "
                                       "attention layer")

    def _check_sandwich_names(self, named):
        """Refuse a checkpoint of the other sandwich_norm kind: one without a sandwich LayerNorm this model has, or
        with one this model does not have (which would otherwise be ignored and leave a different model).  The error
        names the first such variable."""
        want = [rn for i in range(self.L) for rn in self._ref_names(i, True).values() if "/norm_out/" in rn] \
            if self.sandwich_norm else []
        for rn in want:   # layer order: layer_i/attn/norm_out/g, /b, layer_i/mlp/norm_out/g, /b
            if rn not in named:
                raise L.DB200Error(f"load_params: {rn}: missing from the checkpoint of a sandwich_norm model")
        extra = [k for k in named if k.startswith("layer_") and "/norm_out/" in k and k not in want]
        if extra:
            k = min(extra, key=lambda n: (n.split("/")[0], n.split("/")[1] != "attn", n.endswith("/b")))
            raise L.DB200Error(f"load_params: {k}: a sandwich LayerNorm variable, but this model has "
                               f"sandwich_norm = {self.sandwich_norm}")

    def _check_layer_scale_names(self, named):
        """Refuse a checkpoint of the other layer_scale kind: one without a LayerScale vector this model has, or with
        one it does not have.  The error names the first such variable (layer order, the token mixer's first)."""
        want = [rn for i in range(self.L) for k, rn in self._layer_ref_names(i).items() if k in ("lsa", "lsm")]
        for rn in want:
            if rn not in named:
                raise L.DB200Error(f"load_params: {rn}: missing from the checkpoint of a layer_scale model")
        extra = [k for k in named if k.startswith("layer_") and k.endswith("/layer_scale") and k not in want]
        if extra:
            def order(n):   # layer index (a malformed one last), the token mixer's before the MLP's
                i = n.split("/")[0][6:]
                return (int(i) if i.isdigit() else math.inf, n.split("/")[1] == "mlp", n)
            k = min(extra, key=order)
            raise L.DB200Error(f"load_params: {k}: a LayerScale variable, but this model has layer_scale = "
                               f"{self.layer_scale}")

    def _check_position_names(self, named):
        """Refuse a checkpoint of the other position kind: learned positions loaded into a rotary_emb model (which
        would otherwise be ignored), or a rotary_emb checkpoint, which has none, loaded into a model that needs them."""
        wpe = self.EMBED_REF_NAMES["wpe"]
        if self.rotary_emb and wpe in named:
            raise L.DB200Error(f"load_params: {wpe}: a learned position embedding, but this model has rotary_emb = "
                               "true and no learned positions")
        if not self.rotary_emb and wpe not in named:
            raise L.DB200Error(f"load_params: {wpe}: missing from the checkpoint (a rotary_emb checkpoint has no "
                               "learned positions; set rotary_emb to load it)")

    def load_params(self, named):
        """Load a dict keyed by the reference's variable names (SURVEY.md Appendix B); CPU or CUDA fp32 tensors."""
        self.load_flat(self.master, named)
        self.refresh_shadow()

    def _scatter_full(self, name, t, cols=None, rows=None):
        """ZeRO-1: place a full fp32 parameter tensor: bf16 copy (full) + the part of it inside this rank's slice.
        cols / rows: t fills only the first cols columns (a vector: entries) / rows rows of the entry, the rest 0."""
        off, shape = self.layout.entries[name]
        dst16 = self.layout.view(self.shadow, name)
        if cols is None and rows is None and tuple(t.shape) != tuple(shape):
            raise L.DB200Error(f"load_params: {self._ref_embed_name(name)}: expected {tuple(shape)}, got "
                               f"{tuple(t.shape)}")
        if rows is not None and tuple(t.shape) != (rows,) + tuple(shape[1:]):
            raise L.DB200Error(f"load_params: {self._ref_embed_name(name)}: expected {(rows,) + tuple(shape[1:])}, "
                               f"got {tuple(t.shape)}")
        part = lambda x: x[:, :cols] if x.dim() == 2 else x[:cols]   # noqa: E731
        if rows is not None:
            part = lambda x: x[:rows]   # noqa: E731
        elif cols is None:
            part = lambda x: x   # noqa: E731
        part(dst16).copy_(t)
        full = torch.zeros(shape, dtype=F32, device=self.device)
        part(full).copy_(t)
        lo, hi = self.shard
        n = full.numel()
        a, b = max(lo, off), min(hi, off + n)
        if a < b:
            self.master[a - lo:b - lo].copy_(full.view(-1)[a - off:b - off])

    def _refresh_vecs(self):
        """ZeRO-1: rebuild what is derived from the full bf16 parameters (fp32 vector parameters, position table)."""
        ops.gather_cast(self.shadow, self.vec32, self._vec_table, self._vec_table.numel() // 3)
        self._compose_pos()

    def load_flat(self, flat, named):
        """Fill one of the flat fp32 buffers (master | adam_m | adam_v) from a dict of reference-named tensors."""
        dev = self.device
        self._check_sandwich_names(named)
        self._check_layer_kinds(named)
        self._check_layer_scale_names(named)
        self._check_sharing_names(named)
        self._check_position_names(named)
        if self.zero is not None:
            if flat is not self.master:
                raise L.DB200Error("ZeRO-1 mode: loading sharded Adam slots is not implemented (throughput configuration)")
            self.master.zero_(); self.shadow.zero_()
            f32 = lambda x: x.to(device=dev, dtype=F32)
            for name in self.embed_names:
                self._scatter_full(name, f32(named[self._ref_embed_name(name)]),
                                   rows=self.V if name == "wte" and self.tied else None)
            for i in range(self.L):
                p = f"l{i}."
                for k, rn in self._layer_ref_names(i).items():
                    self._scatter_full(p + k, f32(named[rn]))
                if self._is_mlp(i) or not self._owns_mixer(i):
                    continue
                pre = f"layer_{i}/attn/"
                self._scatter_full(p + "wqkv", torch.cat([f32(named[pre + "q"]), f32(named[pre + "k"]),
                                                          f32(named[pre + "v"])], dim=1))
            self._scatter_full("lnf_g", f32(named["to_logits/layer_norm/g"]))
            self._scatter_full("lnf_b", f32(named["to_logits/layer_norm/b"]))
            if not self.tied:
                self._scatter_full("wout", f32(named[self.OUT_KERNEL]), cols=self.V)
            self._scatter_full("bout", f32(named["to_logits/linear_out/bias"]), cols=self.V)
            self._refresh_vecs()
            return
        flat.zero_()
        view = lambda n: self.layout.view(flat, n)

        def put(name, t):
            dst = self.wte_rows(flat) if name == "wte" else view(name)
            t = t.to(device=dev, dtype=F32)
            if tuple(t.shape) != tuple(dst.shape):
                raise L.DB200Error(f"load_params: {self._ref_embed_name(name)}: expected {tuple(dst.shape)}, got "
                                   f"{tuple(t.shape)}")
            dst.copy_(t)

        for name in self.embed_names:
            put(name, named[self._ref_embed_name(name)])
        for i in range(self.L):
            p = f"l{i}."
            ref = self._layer_ref_names(i)
            for k, rn in ref.items():
                put(p + k, named[rn])
            if self._is_mlp(i) or not self._owns_mixer(i):
                continue
            pre = f"layer_{i}/attn/"
            put(p + "wqkv", torch.cat([named[pre + "q"], named[pre + "k"], named[pre + "v"]], dim=1))
        put("lnf_g", named["to_logits/layer_norm/g"]); put("lnf_b", named["to_logits/layer_norm/b"])
        if not self.tied:
            view("wout")[:, :self.V].copy_(named[self.OUT_KERNEL].to(device=dev, dtype=F32))
        view("bout")[:self.V].copy_(named["to_logits/linear_out/bias"].to(device=dev, dtype=F32))

    def export_params(self, source=None):
        """Inverse of load_params: dict of reference-named fp32 CPU tensors (source: master | grads | adam_m | adam_v).
        ZeRO-1: parameters are exported from the full bf16 copy (the reference checkpoints bf16 "master" values under
        bf_16 too, src/dalle_mtf/ops.py:79-80); the sharded Adam slots cannot be exported from one rank."""
        if self.zero is not None and (source is None or source is self.master):
            source = self.shadow
        elif self.zero is not None and source is not self.grads:
            raise L.DB200Error("ZeRO-1 mode: the Adam slots are sharded across ranks")
        flat = self.master if source is None else source
        view = lambda n: (self.wte_rows(flat) if n == "wte" else self.layout.view(flat, n)).detach().float().cpu().clone()
        out = {self._ref_embed_name(n): view(n) for n in self.embed_names}
        d = self.d
        for i in range(self.L):
            p = f"l{i}."
            for k, rn in self._layer_ref_names(i).items():
                out[rn] = view(p + k)
            if self._is_mlp(i) or not self._owns_mixer(i):
                continue
            wqkv = view(p + "wqkv")
            pre = f"layer_{i}/attn/"
            out[pre + "q"], out[pre + "k"], out[pre + "v"] = wqkv[:, :d].clone(), wqkv[:, d:2 * d].clone(), \
                wqkv[:, 2 * d:].clone()
        out["to_logits/layer_norm/g"], out["to_logits/layer_norm/b"] = view("lnf_g"), view("lnf_b")
        if not self.tied:
            out[self.OUT_KERNEL] = view("wout")[:, :self.V].clone()
        out["to_logits/linear_out/bias"] = view("bout")[:self.V].clone()
        return out

    def init_params(self, seed=0):
        """Reference initialisers (SURVEY.md Appendix B), drawn on the device; identical on every rank for a seed."""
        g = torch.Generator(device=self.device).manual_seed(seed)
        d, H, dh, Lyr = self.d, self.H, self.dh, self.L
        if self.zero is not None:
            return self._init_params_sharded(g)
        self.master.zero_()

        def normal(name, std, cols=None, rows=None):
            t = self.P(name)
            if cols is not None:
                t = t[:, :cols] if t.dim() == 2 else t[:cols]
            if rows is not None:
                t = t[:rows]
            t.copy_(torch.randn(t.shape, generator=g, device=self.device, dtype=F32) * std)

        normal("wte", 0.02, rows=self.V)
        if not self.rotary_emb:
            normal("wpe", 0.01)
        if self.row_col:
            normal("image_row", 0.01); normal("image_col", 0.01)
        for i in range(Lyr):
            p = f"l{i}."
            self.P(p + "ln1_g").fill_(1.0); self.P(p + "ln2_g").fill_(1.0)
            if self.sandwich_norm:
                self.P(p + "lna_g").fill_(1.0); self.P(p + "lnm_g").fill_(1.0)
            if self.layer_scale is not None:
                v = layer_scale_init(self.layer_scale, i)
                self.P(p + "lsa").fill_(v); self.P(p + "lsm").fill_(v)
            if not self._owns_mixer(i):   # a shared module is drawn once, at its owner
                pass
            elif self._is_mlp(i):
                w_in, w_sgu, w_out = self._gmlp_init(g, 0.02 / math.sqrt(Lyr))
                self.P(p + "gm_win").copy_(w_in); self.P(p + "sgu_w").copy_(w_sgu); self.P(p + "gm_wout").copy_(w_out)
                self.P(p + "sgu_g").fill_(1.0); self.P(p + "sgu_c").fill_(1.0)
            else:
                wqkv = self.P(p + "wqkv")
                wqkv[:, :d].copy_(torch.randn(d, d, generator=g, device=self.device) * (d ** -0.5 * dh ** -0.5))
                wqkv[:, d:].copy_(torch.randn(d, 2 * d, generator=g, device=self.device) * (d ** -0.5))
                normal(p + "wo", (H * dh) ** -0.5)
            if self._owns_ff(i):
                normal(p + "w1", 0.02)
                normal(p + "w2", 0.02 / math.sqrt(Lyr))
        self.P("lnf_g").fill_(1.0)
        if not self.tied:
            normal("wout", 0.02, cols=self.V)
        self.refresh_shadow()

    def _gmlp_init(self, g, out_std):
        """(W_in, W_sgu, W_out) of a gMLP layer from the generator g, in this order: W_in ~ N(0, 0.02), W_sgu ~
        U(-1e-3 / S, 1e-3 / S) with the strict upper triangle exactly 0 (gMLP's initialisation, so that the block
        starts near h = res with c_sgu = 1), W_out ~ N(0, out_std)."""
        d, S, dev = self.d, self.S, self.device
        w_in = torch.randn(d, 4 * d, generator=g, device=dev, dtype=F32) * 0.02
        eps = 1e-3 / S
        w_sgu = torch.tril((torch.rand(S, S, generator=g, device=dev, dtype=F32) * 2 - 1) * eps)
        w_out = torch.randn(2 * d, d, generator=g, device=dev, dtype=F32) * out_std
        return w_in, w_sgu, w_out

    def _init_params_sharded(self, g):
        """Same initialisers and the same random stream as init_params, one tensor at a time (ZeRO-1: no full fp32 buffer)."""
        d, H, dh, Lyr = self.d, self.H, self.dh, self.L
        self.master.zero_(); self.shadow.zero_()
        rn = lambda shape, std: torch.randn(shape, generator=g, device=self.device, dtype=F32) * std
        ones = lambda n: torch.ones(n, dtype=F32, device=self.device)
        self._scatter_full("wte", rn((self.V, d), 0.02), rows=self.V if self.tied else None)
        for name in self.embed_names[1:]:
            self._scatter_full(name, rn(self.layout.entries[name][1], 0.01))
        for i in range(Lyr):
            p = f"l{i}."
            self._scatter_full(p + "ln1_g", ones(d)); self._scatter_full(p + "ln2_g", ones(d))
            if self.sandwich_norm:
                self._scatter_full(p + "lna_g", ones(d)); self._scatter_full(p + "lnm_g", ones(d))
            if self.layer_scale is not None:
                v = layer_scale_init(self.layer_scale, i)
                self._scatter_full(p + "lsa", ones(d) * v); self._scatter_full(p + "lsm", ones(d) * v)
            if not self._owns_mixer(i):   # a shared module is drawn once, at its owner
                pass
            elif self._is_mlp(i):
                w_in, w_sgu, w_out = self._gmlp_init(g, 0.02 / math.sqrt(Lyr))
                self._scatter_full(p + "gm_win", w_in); self._scatter_full(p + "sgu_w", w_sgu)
                self._scatter_full(p + "gm_wout", w_out)
                self._scatter_full(p + "sgu_g", ones(2 * d)); self._scatter_full(p + "sgu_c", ones(self.S))
            else:
                wq = torch.randn(d, d, generator=g, device=self.device) * (d ** -0.5 * dh ** -0.5)
                wkv = torch.randn(d, 2 * d, generator=g, device=self.device) * (d ** -0.5)
                self._scatter_full(p + "wqkv", torch.cat([wq, wkv], dim=1))
                self._scatter_full(p + "wo", rn((d, d), (H * dh) ** -0.5))
            if self._owns_ff(i):
                self._scatter_full(p + "w1", rn(self.layout.entries[p + "w1"][1], 0.02))
                self._scatter_full(p + "w2", rn((4 * d, d), 0.02 / math.sqrt(Lyr)))
        self._scatter_full("lnf_g", ones(d))
        if not self.tied:
            self._scatter_full("wout", rn((d, self.V), 0.02), cols=self.V)
        self._refresh_vecs()

    def refresh_shadow(self):
        if self.zero is not None:
            return self._refresh_vecs()
        ops.cast_f32_to_bf16(self.master[:self.n_params_padded], self.shadow[:self.n_params_padded])
        self._compose_pos()

    def copy_params_from(self, src):
        """Take over the current weights of `src`, an engine of the same model and rank (evaluation of the weights
        being trained).  ZeRO-1: the fp32 master is only this rank's slice, so the full bf16 copy the kernels read is
        copied too and the fp32 vector parameters are rebuilt from it."""
        self.master.copy_(src.master)
        if self.zero is None:
            return self.refresh_shadow()
        self.shadow.copy_(src.shadow)
        self._refresh_vecs()

    # ------------------------------------------------------------------------------------------ buffers
    def _alloc(self, B):
        key = (B,)
        if self._buf_key == key:
            return self._bufs
        dev, d, S, T = self.device, self.d, self.S, B * self.S
        e = lambda *shape, dtype=BF16: torch.empty(*shape, dtype=dtype, device=dev)
        nt = ops.ce_tiles(self.Vpad)
        n_saved = 1 if self.recompute_grad else self.L
        # token shift: one scratch shared by every layer, the unshifted LayerNorm output in forward and the gradient
        # of the LayerNorm output in backward
        scratch = e(T, d) if self.shift_tokens else None
        raw = {"ln1_raw": scratch, "ln2_raw": scratch} if self.shift_tokens else {}
        # sandwich LayerNorm or LayerScale: both branch outputs (and the statistics of their LayerNorms), for backward
        sand = lambda: self._branch_bufs(T, e)
        # the token mixer's buffers of a saved layer: attention's, a gMLP layer's, or (recompute_grad's one slot) both
        attn_slot = (lambda i: not all(self.mlp)) if self.recompute_grad else (lambda i: not self._is_mlp(i))
        gmlp_slot = (lambda i: any(self.mlp)) if self.recompute_grad else (lambda i: self._is_mlp(i))
        mixer = lambda i: {
            **({"qkv": e(T, 3 * d), "attn": e(T, d), "lse": e(B, self.H, S, dtype=F32)} if attn_slot(i) else {}),
            **(self._gmlp_bufs(T, e, train=True) if gmlp_slot(i) else {})}
        b = {
            "xs": [e(T, d) for _ in range(self.L + 1)],        # residual stream at every layer boundary
            "layers": [{
                "ln1": e(T, d), "mean1": e(T, dtype=F32), "rstd1": e(T, dtype=F32), **mixer(i),
                "xmid": e(T, d), "ln2": e(T, d), "mean2": e(T, dtype=F32), "rstd2": e(T, dtype=F32),
                "h1": e(T, 4 * d), **({"z1": e(T, 4 * d)} if self.gelu else {}),
                **({"z1": e(T, 8 * d)} if self.gated_mlp else {}), **raw, **sand(),
            } for i in range(n_saved)],
            "hf": e(T, d), "meanf": e(T, dtype=F32), "rstdf": e(T, dtype=F32),
            "mf": e(T, dtype=F32) if self.stable else None,   # DivideMax: the rows' maxima
            "labels": e(B, S, dtype=I32), "loss_rows": e(T, dtype=F32),
            # backward scratch
            "dx_a": e(T, d), "dx_b": e(T, d), "dtmp": e(T, d), "dh1": e(T, 4 * d), "dqkv": e(T, 3 * d),
            "delta": e(B, self.H, S, dtype=F32), "dq_acc": e(1, dtype=F32),
        }
        if self.dropout[2] > 0:   # gradient of a branch output before its residual dropout
            b["dxm"] = e(T, d)
        if any(self.mlp):         # gMLP backward: dh (then d gate), dmixed and dgn
            b["g_dh"], b["g_dm"], b["g_dgn"] = e(T, 2 * d), e(T, 2 * d), e(T, 2 * d)
        if self.gated_mlp:        # [dzv | dzg], the gradient of z1
            b["dz1"] = e(T, 8 * d)
        if not self.logits_mask:
            b.update({"part_max": e(nt, T, dtype=F32), "part_sum": e(nt, T, dtype=F32), "label_logit": e(T, dtype=F32),
                      "lse_v": e(T, dtype=F32), "dlogits": e(T, self.Vpad)})
        else:   # one set of vocabulary-product buffers per row block, sized to its window
            b["bias_image"] = e(self.mask_image_cols, dtype=F32)
            b["blocks"] = []
            n_image = B * (S - self.text_rows)
            for rows, N in ((B * self.text_rows, self.mask_text_cols), (n_image, self.mask_image_cols)):
                if rows == 0:   # text_seq_len 1: no text rows
                    b["blocks"].append(None)
                    continue
                nb = ops.ce_tiles(N)
                b["blocks"].append({
                    "rows": rows, "N": N, "hf": e(rows, d), "labels": e(rows, dtype=I32),
                    "part_max": e(nb, rows, dtype=F32), "part_sum": e(nb, rows, dtype=F32),
                    "label_logit": e(rows, dtype=F32), "lse_v": e(rows, dtype=F32), "loss_rows": e(rows, dtype=F32),
                    "dlogits": e(rows, N), "dx": e(rows, d)})
        self._bufs, self._buf_key = b, key
        return b

    def _branch_bufs(self, T, e):
        """The branch outputs oa and om that the sandwich LayerNorm or LayerScale keeps before the residual add, and
        with the sandwich LayerNorm its statistics (nothing without either)."""
        b = {"oa": e(T, self.d), "om": e(T, self.d)} if self.split_branch else {}
        if self.sandwich_norm:
            b.update({"meana": e(T, dtype=F32), "rstda": e(T, dtype=F32), "meanm": e(T, dtype=F32),
                      "rstdm": e(T, dtype=F32)})
        return b

    def _gmlp_bufs(self, T, e, train):
        """A gMLP layer's activations over T rows: res and gate (the two GELU halves of proj_in), gn = LN_sgu(gate) and
        its statistics, h; training also keeps both pre-activations z and mixed for the backward."""
        C = 2 * self.d
        b = {"res": e(T, C), "gate": e(T, C), "gn": e(T, C), "meang": e(T, dtype=F32), "rstdg": e(T, dtype=F32),
             "h": e(T, C)}
        if train:
            b.update({"zres": e(T, C), "zgate": e(T, C), "mixed": e(T, C)})
        return b

    # ------------------------------------------------------------------------------------------ dropout
    def _dropout_descs(self, step, row0):
        """Descriptors of every dropout site for one forward of sequences [row0, row0 + B) of the global batch at
        optimiser step `step` (None where the rate is 0).  Elementwise sites index global token rows row0 * S + t; the
        wpe mask is indexed by position only, so every sequence shares it."""
        emb, att, res = self.dropout
        if step is None or not (emb or att or res):
            return None
        mk = lambda rate, site, r0: L.make_dropout(rate, self.dropout_seed, step, site, r0)
        rows0 = row0 * self.S
        return {
            "wte": mk(emb, L.SITE_WTE, rows0), "wpe": mk(emb, L.SITE_WPE, 0),
            "attn": [mk(att, L.dropout_site_attn(i), row0)
                     if self.radii[i] is None and self.axial[i] is None and (self.conv is None or self.conv[i] is None)
                     and (self.block_sparse is None or self.block_sparse[i] is None) and not self._is_mlp(i) else None
                     for i in range(self.L)],
            "attn_out": [mk(res, L.dropout_site_attn_out(i), rows0) for i in range(self.L)],
            "mlp_out": [mk(res, L.dropout_site_mlp_out(i), rows0) for i in range(self.L)],
        }

    def _site(self, kind, i):
        return self._drop[kind][i] if self._drop is not None else None

    # ------------------------------------------------------------------------------------------ forward
    def _layernorm_fwd(self, x, p, k, sv, S):
        """LayerNorm k (1 or 2) of layer prefix p into sv["ln<k>"]; with the token shift the LayerNorm writes
        sv["ln<k>_raw"] and sv["ln<k>"] receives its shift (rows at position row mod S)."""
        ln = sv[f"ln{k}"]
        out = sv[f"ln{k}_raw"] if self.shift_tokens else ln
        ops.layernorm_fwd(x, self.P(f"{p}ln{k}_g"), self.P(f"{p}ln{k}_b"), out, sv[f"mean{k}"], sv[f"rstd{k}"],
                          self.ln_eps)
        if self.shift_tokens:
            ops.shift_tokens_fwd(out, ln, S, self.text_seq_len, self.shift_w)

    def _branch_out(self, p, norm, x, w, bias, x_res, out, site, sv):
        """The output projection of a branch of layer prefix p and its residual add: out = x_res + drop(x w + bias),
        or with the sandwich LayerNorm sv["o<norm>"] = drop(x w + bias) and out = x_res + LN<norm>(sv["o<norm>"])
        (norm "a": the attention branch's, "m": the MLP's).  LayerScale multiplies what is added by s<norm>."""
        if not self.split_branch:
            return ops.linear_fwd(x, w, out, bias=bias, residual=x_res, dropout=site)
        o = sv["o" + norm]
        ops.linear_fwd(x, w, o, bias=bias, dropout=site)
        self.branch_add(p, norm, o, x_res, out, sv.get("mean" + norm), sv.get("rstd" + norm))

    def branch_add(self, p, norm, o, x_res, out, mean, rstd):
        """The residual add of a stored branch output o (sandwich LayerNorm or LayerScale) of layer prefix p and branch
        norm: out = x_res + v with v = o, or with the sandwich LayerNorm LN<norm>(o) (its statistics into mean / rstd),
        times s<norm> under LayerScale; one rounding.  The decoder's step runs it too."""
        s = self.P(f"{p}ls{norm}") if self.layer_scale is not None else None
        if not self.sandwich_norm:
            return ops.layer_scale_residual_fwd(o, x_res, s, out)
        g, b = self.P(f"{p}ln{norm}_g"), self.P(f"{p}ln{norm}_b")
        if s is None:
            return ops.layernorm_residual_fwd(o, x_res, g, b, out, mean, rstd, self.ln_eps)
        return ops.layernorm_scale_residual_fwd(o, x_res, g, b, s, out, mean, rstd, self.ln_eps)

    def _block_fwd(self, i, x_in, x_out, sv, B, S=None):
        """DALLE.block (src/dalle_mtf/models.py:326-335): x += drop(attn(LN1 x)); x += drop(mlp(LN2 x)); with the
        sandwich LayerNorm x += LNa(drop(attn(LN1 x))); x += LNm(drop(mlp(LN2 x))).
        S: sequence length of the rows (default the model's; prefill runs a shorter prompt)."""
        p = f"l{i}."
        self._layernorm_fwd(x_in, p, 1, sv, S or self.S)
        if self._is_mlp(i):   # gMLP token mixing in place of attention
            self._gmlp_fwd(p, sv, B, S or self.S)
            self._branch_out(p, "a", sv["h"], self.W(p + "gm_wout"), self.P(p + "gm_bout"), x_in, sv["xmid"],
                             self._site("attn_out", i), sv)
        else:
            ops.linear_fwd(sv["ln1"], self.W(p + "wqkv"), sv["qkv"])                   # q|k|v, no bias (:242-244)
            if self.rotary:
                ops.rope_fwd(sv["qkv"], self.rope_table, S or self.S, self.H, self.dh, self.rotary_dim)
            if self.rotary_emb:
                ops.rope_emb_fwd(sv["qkv"], self.rope_emb_table, S or self.S, self.H, self.dh)
            ops.attn_fwd(sv["qkv"], sv["attn"], sv["lse"], B, S or self.S, self.H, self.dh, self.attn_scale,
                         dropout=self._site("attn", i), radius=self.radii[i], **self.axial_kw[i],
                         **self.conv_kw[i], **self.block_sparse_kw[i])  # :257-299
            self._branch_out(p, "a", sv["attn"], self.W(p + "wo"), self.P(p + "o_b"), x_in, sv["xmid"],
                             self._site("attn_out", i), sv)                     # :303-314,330
        self._layernorm_fwd(sv["xmid"], p, 2, sv, S or self.S)
        if self.gated_mlp:   # h1 = zv * act(zg), z1 = [zv | zg] = LN2 W1 + b1 kept for backward (prefill: not written)
            ops.linear_fwd(sv["ln2"], self.W(p + "w1"), sv["h1"], bias=self.P(p + "b1"), glu=self.glu,
                           z_out=sv.get("z1"))
        elif self.gelu:   # h1 = gelu(z1), z1 = LN2 W1 + b1 kept for backward (the prefill's sv has none: not written)
            ops.linear_fwd(sv["ln2"], self.W(p + "w1"), sv["h1"], bias=self.P(p + "b1"), gelu=True,
                           z_out=sv.get("z1"))
        else:
            ops.linear_fwd(sv["ln2"], self.W(p + "w1"), sv["h1"], bias=self.P(p + "b1"), relu=True)     # :320
        self._branch_out(p, "m", sv["h1"], self.W(p + "w2"), self.P(p + "b2"), sv["xmid"], x_out,
                         self._site("mlp_out", i), sv)                          # :321-323,333

    def _gmlp_fwd(self, p, sv, B, n):
        """The token mixing of a gMLP layer over B sequences of n rows: res | gate = gelu(ln1 W_in + b_in) (two GELU
        products, one per half, so that the gate is contiguous for its LayerNorm; z kept when sv has room for it),
        gn = LN_sgu(gate), h = bf16((W_sgu gn + c_sgu) res) (mixed kept likewise)."""
        C = 2 * self.d
        w_in, b_in = self.W(p + "gm_win"), self.P(p + "gm_bin")
        ops.linear_fwd(sv["ln1"], w_in[:, :C], sv["res"], bias=b_in[:C], gelu=True, z_out=sv.get("zres"))
        ops.linear_fwd(sv["ln1"], w_in[:, C:], sv["gate"], bias=b_in[C:], gelu=True, z_out=sv.get("zgate"))
        ops.layernorm_fwd(sv["gate"], self.P(p + "sgu_g"), self.P(p + "sgu_b"), sv["gn"], sv["meang"], sv["rstdg"],
                          self.ln_eps)
        ops.sgu_mix_fwd(self.W(p + "sgu_w"), sv["gn"], sv["res"], self.P(p + "sgu_c"), sv["h"], sv.get("mixed"), B, n)

    def ce_weights(self, global_batch):
        """lib.CeWeights of the weighted loss for a step over `global_batch` sequences (all ranks and micro-batches)."""
        a_text, a_image = loss_coefficients(self.loss_weights, self.text_seq_len, self.image_seq_len, global_batch)
        return L.make_ce_weights(self.S, self.text_seq_len - 1, a_text, a_image, self.z_loss)

    def loss_part_scales(self, global_batch):
        """Factors that turn the sums [1..3] of a weighted forward into the text-row mean CE, the image-row mean CE
        and the mean z-term over all rows."""
        n_text = max(self.text_seq_len - 1, 1)
        return 1.0 / (global_batch * n_text), 1.0 / (global_batch * (self.image_seq_len + 1)), \
            1.0 / (global_batch * self.S)

    def forward(self, tokens, loss_accum=None, step=None, row0=0, global_batch=None):
        """tokens int32 [B,S] on the device.  Adds sum_t loss_rows[t] of this batch into the 1-element fp32 tensor
        `loss_accum` (default: the aux slot behind the gradients, which rides along with the gradient all-reduce)
        and returns it.  The mean over all positions (src/dalle_mtf/models.py:353-354) is that sum / (global B*S).

        Weighted loss (loss_weights / z_loss): loss_rows[t] = CE_t + z lse_t^2 and loss_accum (4 floats, default aux
        slots 0-3) receives (sum_t a_t loss_rows[t], text-row CE sum, image-row CE sum, z-term sum), with the
        coefficients a_t of a step over `global_batch` sequences (default B): slot 0 then is this batch's share of the
        loss itself.

        step: the global optimiser step of a training forward; with a step the dropout rates apply (mode "train"),
        without one they do not.  row0: global index of tokens[0] in the step's batch (rank and micro-batch offset),
        so that the masks do not depend on how the batch is split."""
        B, S = tokens.shape
        assert S == self.S, f"expected sequence length {self.S}, got {S}"
        bufs = self._alloc(B)
        T = B * S
        self._tokens = tokens
        self._drop = self._dropout_descs(step, row0)
        if self._drop is not None:
            ops.embed_fwd(tokens, self.embed_table(), self.pos_embedding(), bufs["xs"][0].view(B, S, self.d),
                          wte_drop=self._drop["wte"], wpe_drop=self._drop["wpe"])            # models.py:198-217
        else:
            ops.embed_fwd(tokens, self.embed_table(), self.pos_embedding(),
                          bufs["xs"][0].view(B, S, self.d))                                   # models.py:399
        for i in range(self.L):
            sv = bufs["layers"][0 if self.recompute_grad else i]
            self._block_fwd(i, bufs["xs"][i], bufs["xs"][i + 1], sv, B)
        self.final_ln(bufs["xs"][self.L], bufs["hf"], bufs["meanf"], bufs["rstdf"], bufs["mf"])  # models.py:393
        ops.shift_labels(tokens, bufs["labels"], self.eos_token_id)                                # models.py:407-410
        labels = bufs["labels"].view(T)
        if self.logits_mask:
            return self._masked_forward(bufs, B, loss_accum, global_batch)
        self.vocab_gemm(bufs["hf"], None, mode=L.EPI_CE_STATS, bias=self.P("bout"), labels=labels,
                        part_max=bufs["part_max"], part_sum=bufs["part_sum"], label_logit=bufs["label_logit"],
                        n_valid=self.V)
        if self.weighted_loss:
            self._cew = self.ce_weights(B if global_batch is None else global_batch)
            if loss_accum is None:
                loss_accum = self.grads[self.aux_off:self.aux_off + 4]
            ops.ce_finish_weighted(bufs["part_max"], bufs["part_sum"], bufs["label_logit"], bufs["lse_v"],
                                   bufs["loss_rows"], loss_accum, self._cew)
            return loss_accum
        if loss_accum is None:
            loss_accum = self.grads[self.aux_off:self.aux_off + 1]
        ops.ce_finish(bufs["part_max"], bufs["part_sum"], bufs["label_logit"], bufs["lse_v"], bufs["loss_rows"],
                      loss_accum)
        return loss_accum

    def final_ln(self, x, hf, mean, rstd, m):
        """hf = LN_f(x) (statistics into mean / rstd); with `stable` LN_f(x / max(x)) per row, the maxima into m.  The
        prefill and the decoder's step run it too."""
        if self.stable:
            return ops.layernorm_divmax_fwd(x, self.P("lnf_g"), self.P("lnf_b"), hf, mean, rstd, m, self.ln_eps)
        return ops.layernorm_fwd(x, self.P("lnf_g"), self.P("lnf_b"), hf, mean, rstd, self.ln_eps)

    # ------------------------------------------------------------------------------------------ logits mask
    def _mask_windows(self):
        """(first column, n_valid) of the text and the image block's vocabulary window; the image block's labels are
        relative to its first column."""
        c0 = self.mask_c0
        return ((0, self.image_offset), (c0, self.V - c0))

    def _masked_forward(self, bufs, B, loss_accum, global_batch):
        """The vocabulary products of forward() with the logits mask: partition hf and the labels into the text and
        image blocks, CE_STATS + finish on each block over its window (text block first: fixed order), scatter the
        row losses back into [B*S] order."""
        S, d = self.S, self.d
        text, image = bufs["blocks"]
        ops.logits_mask_partition(bufs["hf"], bufs["labels"].view(-1), self.P("bout"),
                                  text["hf"] if text else None, image["hf"], text["labels"] if text else None,
                                  image["labels"], bufs["bias_image"], B, S, self.text_rows, self.mask_c0,
                                  self.image_offset, self.V)
        if self.weighted_loss:
            a_text, a_image = loss_coefficients(self.loss_weights, self.text_seq_len, self.image_seq_len,
                                                B if global_batch is None else global_batch)
            self._cew = (L.make_ce_weights(1, 1, a_text, a_image, self.z_loss),
                         L.make_ce_weights(1, 0, a_text, a_image, self.z_loss))
            if loss_accum is None:
                loss_accum = self.grads[self.aux_off:self.aux_off + 4]
        elif loss_accum is None:
            loss_accum = self.grads[self.aux_off:self.aux_off + 1]
        biases = (self.P("bout"), bufs["bias_image"])
        for k, ((c0, n_valid), blk) in enumerate(zip(self._mask_windows(), bufs["blocks"])):
            if blk is None:
                continue
            self.vocab_gemm(blk["hf"], None, c0, blk["N"], mode=L.EPI_CE_STATS, bias=biases[k], labels=blk["labels"],
                            part_max=blk["part_max"], part_sum=blk["part_sum"], label_logit=blk["label_logit"],
                            n_valid=n_valid)
            if self.weighted_loss:
                ops.ce_finish_weighted(blk["part_max"], blk["part_sum"], blk["label_logit"], blk["lse_v"],
                                       blk["loss_rows"], loss_accum, self._cew[k])
            else:
                ops.ce_finish(blk["part_max"], blk["part_sum"], blk["label_logit"], blk["lse_v"], blk["loss_rows"],
                              loss_accum)
        ops.logits_mask_scatter(B, S, self.text_rows, loss_text=text["loss_rows"] if text else None,
                                loss_image=image["loss_rows"], loss_rows=bufs["loss_rows"])
        return loss_accum

    def _masked_backward(self, bufs, B, grad_scale):
        """The vocabulary products of backward() with the logits mask: per block (text first) the CE_GRAD product with
        its fused bias gradient, the wout wgrad and the dgrad, all over the block's window and accumulating into
        G("wout") / G("bout") at its column offset; then the two dgrads are scattered into bufs["dtmp"]."""
        d = self.d
        biases = (self.P("bout"), bufs["bias_image"])
        for k, ((c0, n_valid), blk) in enumerate(zip(self._mask_windows(), bufs["blocks"])):
            if blk is None:
                continue
            N = blk["N"]
            cew = None
            if self.weighted_loss:
                c = self._cew[k]
                cew = L.make_ce_weights(c.period, c.text_rows, c.a_text * grad_scale, c.a_image * grad_scale, c.z_loss)
            self.vocab_gemm(blk["hf"], blk["dlogits"], c0, N, mode=L.EPI_CE_GRAD, alpha=grad_scale, bias=biases[k],
                            labels=blk["labels"], lse=blk["lse_v"], n_valid=n_valid, colsum=self.G("bout")[c0:c0 + N],
                            ce_weights=cew)
            self.vocab_wgrad(blk["hf"], blk["dlogits"], c0, N)
            self.vocab_dgrad(blk["dlogits"], blk["dx"], c0, N)
        text, image = bufs["blocks"]
        ops.logits_mask_scatter(B, self.S, self.text_rows, dx_text=text["dx"] if text else None, dx_image=image["dx"],
                                dx=bufs["dtmp"])

    def logits(self, tokens):
        """fp32 logits [B,S,V] (return_logits=True path, src/dalle_mtf/models.py:412-415).  Test / eval use only:
        this materialises the tensor the training path never writes.  With the logits mask, -inf outside each row's
        window, so that softmax(logits) is the model's distribution."""
        B, S = tokens.shape
        self.forward(tokens, loss_accum=torch.zeros(4 if self.weighted_loss else 1, dtype=F32, device=self.device))
        T = B * S
        out = torch.empty(T, self.Vpad, dtype=F32, device=self.device)
        self.vocab_gemm(self._bufs["hf"], out, bias=self.P("bout"))
        logits = out.view(B, S, self.Vpad)[:, :, :self.V]
        if self.logits_mask:
            logits[:, :self.text_rows, self.image_offset:] = -math.inf
            logits[:, self.text_rows:, :self.image_offset] = -math.inf
        return logits

    # ------------------------------------------------------------------------------------------ prompt prefill
    def _prefill_alloc(self, B, P, rep):
        """Compact buffers of one prefill: B*P rows, shared by every layer (nothing is kept for a backward pass)."""
        key = (B, P, rep)
        if getattr(self, "_pf_key", None) == key:
            return self._pf
        dev, d, T = self.device, self.d, B * P
        e = lambda *shape, dtype=BF16: torch.empty(*shape, dtype=dtype, device=dev)
        self._pf = {
            "xs": [e(T, d), e(T, d)],
            "sv": {"ln1": e(T, d), "mean1": e(T, dtype=F32), "rstd1": e(T, dtype=F32), "qkv": e(T, 3 * d),
                   "attn": e(T, d), "lse": e(B, self.H, P, dtype=F32), "xmid": e(T, d), "ln2": e(T, d),
                   "mean2": e(T, dtype=F32), "rstd2": e(T, dtype=F32), "h1": e(T, 4 * d),
                   # token shift: both unshifted LayerNorm outputs stay until the layer's caches are filled
                   **({"ln1_raw": e(T, d), "ln2_raw": e(T, d)} if self.shift_tokens else {}),
                   # sandwich LayerNorm or LayerScale: the branch outputs (and their LayerNorms' statistics)
                   **self._branch_bufs(T, e),
                   # gMLP layers: their activations without what only a backward reads
                   **(self._gmlp_bufs(T, e, train=False) if any(self.mlp) else {})},
            "x_last": e(B * rep, d), "hf": e(B * rep, d), "meanf": e(B * rep, dtype=F32),
            "rstdf": e(B * rep, dtype=F32), "logits": e(B * rep, self.Vpad, dtype=F32),
            "mf": e(B * rep, dtype=F32) if self.stable else None,
        }
        self._pf_key = key
        return self._pf

    def prefill(self, tokens, k_caches, v_caches, rep=1, shift_caches=None):
        """Runs a whole prompt, tokens int32 [B, P] (1 <= P < S), through the training forward kernels in one pass
        and hands it to the decoder: every layer's k / v of positions < P go into k_caches[i] / v_caches[i] (bf16
        [B*rep, S, H, dh], rows b*rep .. b*rep + rep - 1 all receive prompt b), and the result is the fp32 logits
        [B*rep, Vpad] of position P for each replica.  No dropout (inference); the training buffers and the state a
        pending backward() reads are left untouched.

        shift_caches (required with the token shift, else None): 2 L bf16 [B*rep, S, d/2] caches, layer i's LN1 at
        2i and its LN2 at 2i + 1; positions < P receive the first d/2 columns of the unshifted LayerNorm outputs.

        A gMLP layer i has no k / v: k_caches[i] is its bf16 [B*rep, S, 2d] cache of the SGU LayerNorm outputs gn
        (positions < P filled, same replica order) and v_caches[i] is None."""
        B, P = tokens.shape
        if not 1 <= P < self.S:
            raise ValueError(f"prefill: prompt length {P} outside [1, {self.S})")
        if int(rep) != rep or rep < 1:
            raise ValueError(f"prefill: rep must be an integer >= 1, got {rep!r}")
        rep = int(rep)
        shape = (B * rep, self.S, self.H, self.dh)
        gshape = (B * rep, self.S, 2 * self.d)
        if len(k_caches) != self.L or len(v_caches) != self.L or \
                any((tuple(k.shape) != gshape or v is not None) if m else
                    (k is None or v is None or tuple(k.shape) != shape or tuple(v.shape) != shape)
                    for k, v, m in zip(k_caches, v_caches, [self._is_mlp(i) for i in range(self.L)])):
            raise ValueError(f"prefill: expected {self.L} k and v caches of shape {shape} (a gMLP layer: its SGU cache "
                             f"{gshape} and None)")
        if self.shift_tokens:
            sshape = (B * rep, self.S, self.d // 2)
            if shift_caches is None or len(shift_caches) != 2 * self.L or \
                    any(tuple(c.shape) != sshape for c in shift_caches):
                raise ValueError(f"prefill: the token shift needs {2 * self.L} shift caches of shape {sshape}")
        elif shift_caches is not None:
            raise ValueError("prefill: shift_caches given to an engine without the token shift")
        b = self._prefill_alloc(B, P, rep)
        d = self.d
        ops.embed_fwd(tokens, self.embed_table(), self.pos_embedding(), b["xs"][0].view(B, P, d))
        drop, self._drop = self._drop, None        # restored below: backward() of a preceding forward() reads it
        try:
            x_in, x_out = b["xs"]
            for i in range(self.L):
                self._block_fwd(i, x_in, x_out, b["sv"], B, S=P)
                if self._is_mlp(i):
                    ops.sgu_cache_fill(b["sv"]["gn"], k_caches[i], P, rep)
                else:
                    ops.kv_cache_fill(b["sv"]["qkv"], k_caches[i], v_caches[i], P, rep)
                if self.shift_tokens:
                    ops.shift_cache_fill(b["sv"]["ln1_raw"], shift_caches[2 * i], P, rep)
                    ops.shift_cache_fill(b["sv"]["ln2_raw"], shift_caches[2 * i + 1], P, rep)
                x_in, x_out = x_out, x_in
        finally:
            self._drop = drop
        ops.rows_repeat(x_in.view(B, P, d)[:, P - 1], b["x_last"], rep)
        self.final_ln(b["x_last"], b["hf"], b["meanf"], b["rstdf"], b["mf"])
        self.vocab_gemm(b["hf"], b["logits"], bias=self.P("bout"))
        return b["logits"]

    # ------------------------------------------------------------------------------------------ backward
    def _ln_bwd(self, dy, x, g, mean, rstd, dres, dx, dg, db, dxsum, site, m=None):
        """LayerNorm backward; when `site` (the residual-dropout site of the branch whose output x sums) is active it
        also writes bufs["dxm"] = dx * keep * scale, and dxsum is colsum(dxm).  Returns the gradient of that branch
        output (dxm, or dx without dropout).  m: the rows' maxima of a DivideMax LayerNorm (final_ln with `stable`)."""
        if m is not None:
            dxm = None if site is None else self._bufs["dxm"]
            ops.layernorm_divmax_bwd(dy, x, g, mean, rstd, m, dres, dx, dg, db, dxsum=dxsum, dxm=dxm, dropout=site)
            return dx if dxm is None else dxm
        if site is None:
            ops.layernorm_bwd(dy, x, g, mean, rstd, dres, dx, dg, db, dxsum=dxsum)
            return dx
        dxm = self._bufs["dxm"]
        ops.layernorm_bwd(dy, x, g, mean, rstd, dres, dx, dg, db, dxsum=dxsum, dxm=dxm, dropout=site)
        return dxm

    def _shift_bwd(self, dshifted, out):
        """The token shift's transpose: the gradient of the unshifted LayerNorm output, written to `out`."""
        ops.shift_tokens_bwd(dshifted, out, self.S, self.text_seq_len, self.shift_w)
        return out

    def _block_bwd(self, i, x_in, sv, dx_out, dx_in, bufs, B, dxsum_below, dbranch):
        """Backward of one block.  Bias gradients are column sums of activation gradients; they are produced by the
        kernel that WRITES that gradient (LayerNorm-backward / ReLU-mask epilogue) instead of separate passes:
        db2 (= colsum of this block's output gradient) was already accumulated by whoever produced dx_out.
        dbranch: gradient of the MLP output before its residual dropout (dx_out itself without dropout).  Returns the
        same for the layer below.

        Sandwich LayerNorm or LayerScale (split_branch): the branch gradients come from _branch_bwd on dx_out and on
        dx_mid, which fuses their dropout and the b2 / o_b column sums, so dbranch and dxsum_below are None and the
        LayerNorms that produce dx_mid and dx_in fuse neither.  dx_in may be dx_out's storage: the token mixer's branch
        gradient goes there once dx_out is consumed, and LN1's backward overwrites it last."""
        p = f"l{i}."
        split = self.split_branch
        ob = p + ("gm_bout" if self._is_mlp(i) else "o_b")   # the token mixer's output bias
        if split:   # dbranch = d om * keep * scale, db2 = colsum(dbranch)
            dbranch = self._branch_bwd(p, "m", dx_out, sv, bufs, bufs["dtmp"], self.G(p + "b2"),
                                       self._site("mlp_out", i))
        # ---- MLP
        dz = bufs["dz1"] if self.gated_mlp else bufs["dh1"]   # the gradient of W1's output
        if self.gated_mlp:   # dh = dx W2^T -> dz1 = [dh a | dh act'(zg) zv]; db1 = colsum(dz1)
            ops.linear_dgrad(dbranch, self.W(p + "w2"), dz, glu_grad_of=sv["z1"], glu=self.glu, colsum=self.G(p + "b1"))
        elif self.gelu:   # dZ = (dx W2^T) * gelu'(z1); db1
            ops.linear_dgrad(dbranch, self.W(p + "w2"), bufs["dh1"], gelu_grad_of=sv["z1"], colsum=self.G(p + "b1"))
        else:
            ops.linear_dgrad(dbranch, self.W(p + "w2"), bufs["dh1"], relu_mask_of=sv["h1"],
                             colsum=self.G(p + "b1"))                                   # dH = (dx W2^T)*[h1>0]; db1
        ops.linear_wgrad(sv["h1"], dbranch, self.G(p + "w2"))
        ops.linear_dgrad(dz, self.W(p + "w1"), bufs["dtmp"])                                  # dLN2 out
        ops.linear_wgrad(sv["ln2"], dz, self.G(p + "w1"))
        dln = self._shift_bwd(bufs["dtmp"], sv["ln2_raw"]) if self.shift_tokens else bufs["dtmp"]
        dx_mid = bufs["dx_b"] if dx_out is bufs["dx_a"] else bufs["dx_a"]
        da = self._ln_bwd(dln, sv["xmid"], self.P(p + "ln2_g"), sv["mean2"], sv["rstd2"], dx_out, dx_mid,
                          self.G(p + "ln2_g"), self.G(p + "ln2_b"), None if split else self.G(ob),
                          None if split else self._site("attn_out", i))                 # do_b = colsum(da)
        if split:   # da = d oa * keep * scale, do_b = colsum(da)
            da = self._branch_bwd(p, "a", dx_mid, sv, bufs, dx_in, self.G(ob), self._site("attn_out", i))
        if self._is_mlp(i):   # ---- gMLP token mixing
            self._gmlp_bwd(p, sv, da, bufs, B)
        else:             # ---- attention
            ops.linear_dgrad(da, self.W(p + "wo"), bufs["dtmp"])                              # d(attn out)
            ops.linear_wgrad(sv["attn"], da, self.G(p + "wo"))
            ops.attn_bwd(sv["qkv"], sv["attn"], bufs["dtmp"], sv["lse"], bufs["dq_acc"], bufs["delta"], bufs["dqkv"],
                         B, self.S, self.H, self.dh, self.attn_scale, dropout=self._site("attn", i),
                         radius=self.radii[i], **self.axial_kw[i], **self.conv_kw[i], **self.block_sparse_kw[i])
            if self.rotary:   # d(q|k|v) before the rotation
                ops.rope_bwd(bufs["dqkv"], self.rope_table, self.S, self.H, self.dh, self.rotary_dim)
            if self.rotary_emb:
                ops.rope_emb_bwd(bufs["dqkv"], self.rope_emb_table, self.S, self.H, self.dh)
            ops.linear_dgrad(bufs["dqkv"], self.W(p + "wqkv"), bufs["dtmp"])                  # dLN1 out
            ops.linear_wgrad(sv["ln1"], bufs["dqkv"], self.G(p + "wqkv"))
        dln = self._shift_bwd(bufs["dtmp"], sv["ln1_raw"]) if self.shift_tokens else bufs["dtmp"]
        return self._ln_bwd(dln, x_in, self.P(p + "ln1_g"), sv["mean1"], sv["rstd1"], dx_mid, dx_in,
                            self.G(p + "ln1_g"), self.G(p + "ln1_b"), dxsum_below,
                            self._site("mlp_out", i - 1) if i > 0 and not split else None)   # db2 of the layer below

    def _branch_bwd(self, p, norm, dy, sv, bufs, out, dbias, site):
        """The gradient of branch output o<norm> of layer prefix p before its residual dropout `site`, from dy, the
        gradient of the residual sum it was added to: into `out` (bufs["dxm"] with dropout under the sandwich
        LayerNorm), with dbias += its column sum.  LayerScale: d(s<norm>) += colsum(dy v) and the scaled gradient is
        s dy; with the sandwich LayerNorm that goes through a [T, d] prefix of bufs["dh1"] (free until the MLP's
        dgrad writes it) into LN<norm>'s backward."""
        if self.layer_scale is not None:
            s, ds = self.P(f"{p}ls{norm}"), self.G(f"{p}ls{norm}")
            if not self.sandwich_norm:
                return ops.layer_scale_bwd(dy, sv["o" + norm], s, out, ds, db=dbias, dropout=site)
            dv = bufs["dh1"].view(-1)[:dy.numel()].view(dy.shape)
            ops.layer_scale_bwd(dy, sv["o" + norm], s, dv, ds, norm=(self.P(f"{p}ln{norm}_g"), self.P(f"{p}ln{norm}_b"),
                                                                     sv["mean" + norm], sv["rstd" + norm]))
            dy = dv
        return self._ln_bwd(dy, sv["o" + norm], self.P(f"{p}ln{norm}_g"), sv["mean" + norm], sv["rstd" + norm], None,
                            out, self.G(f"{p}ln{norm}_g"), self.G(f"{p}ln{norm}_b"), dbias, site)

    def _gmlp_bwd(self, p, sv, da, bufs, B):
        """Backward of a gMLP layer's token mixing from da, the gradient of the branch output before its bias: into
        bufs["dtmp"] (the gradient of the LN1 output) and the layer's W_out, c_sgu, W_sgu, SGU norm, W_in and b_in
        gradients.  du = [du_res | du_gate] is formed in bufs["dh1"] (free once the MLP branch is done)."""
        C, S = 2 * self.d, self.S
        dh, dm, dgn, du = bufs["g_dh"], bufs["g_dm"], bufs["g_dgn"], bufs["dh1"]
        ops.linear_dgrad(da, self.W(p + "gm_wout"), dh)                                      # dh
        ops.linear_wgrad(sv["h"], da, self.G(p + "gm_wout"))
        # dmixed = dh res, du_res = dh mixed gelu'(z_res), dc_sgu
        ops.sgu_bwd(dh, sv["mixed"], sv["res"], sv["zres"], dm, du[:, :C], self.G(p + "sgu_c"), B, S)
        ops.sgu_mix_dgrad(self.W(p + "sgu_w"), dm, dgn, B, S)                                # dgn = W^T dmixed
        ops.sgu_mix_wgrad(dm, sv["gn"], self.G(p + "sgu_w"), B, S)                           # dW (lower triangle)
        ops.layernorm_bwd(dgn, sv["gate"], self.P(p + "sgu_g"), sv["meang"], sv["rstdg"], None, dh,
                          self.G(p + "sgu_g"), self.G(p + "sgu_b"))                          # d gate (into dh)
        ops.sgu_gate_bwd(dh, sv["zgate"], du[:, C:])                                        # du_gate
        ops.colsum(du, self.G(p + "gm_bin"))                                                 # db_in
        ops.linear_dgrad(du, self.W(p + "gm_win"), bufs["dtmp"])                             # dLN1 out
        ops.linear_wgrad(sv["ln1"], du, self.G(p + "gm_win"))

    def backward(self, grad_scale, on_bucket_ready=None):
        """Back-propagates d(sum(loss_rows) * grad_scale); with the weighted loss d(sum_t a_t loss_rows[t] * grad_scale)
        (the coefficients of the preceding forward).  Gradients ACCUMULATE into self.grads.
        on_bucket_ready(start, end) is called as soon as the flat range [start, end) is final (data-parallel hook)."""
        bufs = self._bufs
        tokens = self._tokens
        B, S = tokens.shape
        T, d = B * S, self.d
        if self.logits_mask:
            self._masked_backward(bufs, B, grad_scale)
        else:
            labels = bufs["labels"].view(T)
            cew = None
            if self.weighted_loss:
                c = self._cew
                cew = L.make_ce_weights(c.period, c.text_rows, c.a_text * grad_scale, c.a_image * grad_scale, c.z_loss)
            self.vocab_gemm(bufs["hf"], bufs["dlogits"], mode=L.EPI_CE_GRAD, alpha=grad_scale, bias=self.P("bout"),
                            labels=labels, lse=bufs["lse_v"], n_valid=self.V, colsum=self.G("bout"),
                            ce_weights=cew)  # dlogits + fused d(bout) = colsum(dlogits)
            self.vocab_wgrad(bufs["hf"], bufs["dlogits"])
            self.vocab_dgrad(bufs["dlogits"], bufs["dtmp"])
        dx = bufs["dx_a"]
        split = self.split_branch   # the branch's own backward fuses db2 and the mlp_out dropout instead
        dbranch = self._ln_bwd(bufs["dtmp"], bufs["xs"][self.L], self.P("lnf_g"), bufs["meanf"], bufs["rstdf"], None,
                               dx, self.G("lnf_g"), self.G("lnf_b"), None if split else self.G(f"l{self.L - 1}.b2"),
                               None if split else self._site("mlp_out", self.L - 1),    # db2 of the last block
                               bufs["mf"])
        if on_bucket_ready:
            s, e = self.layout.span("lnf_g", "bout")
            on_bucket_ready(s, e + 64)  # + the aux scalars (loss) that sit behind the last parameter
        for i in reversed(range(self.L)):
            if self.recompute_grad:  # mtf.recompute_grad per block, src/dalle_mtf/models.py:342-343
                sv = bufs["layers"][0]
                self._block_fwd(i, bufs["xs"][i], bufs["dtmp"], sv, B)
            else:
                sv = bufs["layers"][i]
            # dx (grad w.r.t. the block output) is dead once dx_mid has been formed in the other buffer, so the
            # block's input gradient is written back into the same storage.
            dbranch = self._block_bwd(i, bufs["xs"][i], sv, dx, dx, bufs, B,
                                      self.G(f"l{i - 1}.b2") if i > 0 and not split else None, dbranch)
            if on_bucket_ready:
                s, e = self.layout.span(f"l{i}.ln1_g", self.layer_last(i))
                on_bucket_ready(s, e)
        # row / column positions: the gradient of the composed table goes into a zeroed scratch, then is folded into
        # wpe, image_row and image_col (one fully formed contribution per call, like the wpe gradient itself)
        # (rotary_emb: the zero table's gradient goes to the scratch and is not read)
        dpos = self._dpos.zero_() if self.row_col or self.rotary_emb else self.G("wpe")
        dwte = self.wte_rows(self.grads)   # tied: after the vocabulary wgrad, in this fixed order
        alpha = {"alpha": STABLE_ALPHA} if self.stable else {}   # pos_fold is linear: it carries the shrink along
        if self._drop is not None:
            ops.embed_bwd(tokens, dx.view(B, S, d), dwte, dpos, wte_drop=self._drop["wte"],
                          wpe_drop=self._drop["wpe"], **alpha)
        else:
            ops.embed_bwd(tokens, dx.view(B, S, d), dwte, dpos, **alpha)
        if self.row_col:
            ops.pos_fold(dpos, self.G("wpe"), self.G("image_row"), self.G("image_col"))
        if on_bucket_ready:
            s, e = self.layout.span("wte", self.embed_names[-1])
            on_bucket_ready(s, e)

    # ------------------------------------------------------------------------------------------ optimiser
    def zero_grads(self):
        """Gradients accumulate (+=), so every step starts from zeros.  The Adam kernel writes those zeros while it
        streams the gradient it consumes, so after an optimiser step only the 64 aux scalars (loss) need clearing; the
        full 4 B/param memset runs only when backward ran without an optimiser step in between (tests, first step)."""
        if self._grads_clean:
            self.grads[self.aux_off:].zero_()
        else:
            self.grads.zero_()
        self._grads_clean = False

    def _decay_segments(self):
        """Contiguous [start, end, decays) runs of the flat buffer: mtf's AdamWeightDecayOptimizer is built with
        exclude_from_weight_decay=["norm", "bias"] (src/optimizers.py:84-88), i.e. every variable whose NAME contains
        "norm" or "bias" (LayerNorm g/b, all biases incl. compute_output_bias/o_b) is left undecayed."""
        if getattr(self, "_segs", None) is None:
            decays = lambda n: n in ("wte", "wpe", "image_row", "image_col", "wout") or \
                n.split(".")[-1] in ("wqkv", "wo", "w1", "w2", "gm_win", "sgu_w", "gm_wout")
            segs = []
            for name in self.layout.order:
                s, e = self.layout.span(name, name)
                d = decays(name)
                if segs and segs[-1][2] == d and segs[-1][1] == s:
                    segs[-1][1] = e
                else:
                    segs.append([s, e, d])
            self._segs = [tuple(x) for x in segs]
        return self._segs

    def optimizer_step(self, lr, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.0, clip=1.0):
        """clip_by_global_norm + mtf AdamWeightDecayOptimizer (src/optimizers.py:11-16, 82-103); no host sync.
        clip=None disables clipping (explicit `"gradient_clipping": null`, optimizers.py:101)."""
        n = self.n_params_padded
        if clip and clip > 0:
            self.gnorm_sq.zero_()
            ops.sqnorm(self.grads[:n], self.gnorm_sq)       # the reduced gradient is identical on every rank
            gn = self.gnorm_sq
        else:
            gn, clip = None, 0.0
        if self.zero is not None:
            if weight_decay:
                raise L.DB200Error("ZeRO-1 mode: weight_decay != 0 is not wired (no reference config uses it)")
            lo, hi = self.shard
            m = hi - lo
            if m > 0:   # this rank's slice: fp32 master + Adam slots, bf16 result written into the full copy
                ops.adam_step(self.master[:m], self.adam_m[:m], self.adam_v[:m], self.grads[lo:hi], self.shadow[lo:hi],
                              lr, beta1, beta2, eps, 0.0, gn, clip, 1.0, False, 0)
            self.zero.all_gather_inplace(self.shadow, self.chunk)   # bf16 parameters of every slice
            self._refresh_vecs()
            return
        if not weight_decay:
            ops.adam_step(self.master[:n], self.adam_m[:n], self.adam_v[:n], self.grads[:n], self.shadow[:n], lr,
                          beta1, beta2, eps, 0.0, gn, clip, 1.0, False, 0, zero_grad=True)
            self._grads_clean = True
            return self._compose_pos()
        for s, e, d in self._decay_segments():     # `update += weight_decay * param` only on the kernels / embeddings
            ops.adam_step(self.master[s:e], self.adam_m[s:e], self.adam_v[s:e], self.grads[s:e], self.shadow[s:e], lr,
                          beta1, beta2, eps, weight_decay if d else 0.0, gn, clip, 1.0, False, 0)
        self._compose_pos()
