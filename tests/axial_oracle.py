"""Float64 / fp32 reference of DALL-E transformers with axial (row and column) attention layers, for the tests.

Axial layers are an extension, not in the reference: DALL-E's row and column attention, DALLE-pytorch's "axial_row"
and "axial_col".  With TL = text_seq_len and the image tokens on a W x W grid (image_seq_len = W^2), position p >= TL
is the image token at row r = (p - TL) // W, column c = (p - TL) % W.  Text queries are causal, as in a global layer.
An image query sees every text key plus, in a row layer, the image keys of row r at columns <= c and, in a column
layer, those of column c at rows <= r.  The mask is built here from (r, c) in the original order; the kernels walk a
column layer's image rows column-major instead (dalle_mtf_b200/csrc/attn_fa.cu).  Axial layers get no attention
dropout (the dropout site 2 + 3l of an axial layer l is unused) and keep their residual dropout.

Global and local layers take oracle.dalle_local's masks, and forward() is oracle.dalle_local.forward operation for
operation, so a model without axial layers computes bit for bit what that module computes.
"""
import math
from dataclasses import dataclass

import torch

from oracle import dalle_local as OL
from oracle.dalle import Quirks, _r, layer_norm, shift_labels

AXES = {"axial_row": 0, "axial_col": 1}


@dataclass
class AxialConfig(OL.LocalConfig):
    """oracle.dalle_local.LocalConfig whose attention_types may also hold "axial_row" / "axial_col"."""

    def is_axial(self, layer):
        return self.attention_types is not None and self.attention_types[layer] in AXES

    @property
    def grid_w(self):
        """Width W of the image-token grid, image_seq_len = W^2."""
        W = math.isqrt(self.image_seq_len)
        if W * W != self.image_seq_len:
            raise ValueError(f"axial attention needs a square image_seq_len, got {self.image_seq_len}")
        return W


def axial_hidden(S, text_len, grid_w, axis, shift=0):
    """[S,S] bool: True where query i may not see key j in an axial layer.  shift moves every image key's row (axis 0)
    or column (axis 1) index by `shift` before it is compared with the query's: a deliberately wrong mask whose
    segment is off by one, for the edge tests."""
    i = torch.arange(S)[:, None]
    j = torch.arange(S)[None, :]
    ki, kj = i - text_len, j - text_len
    if axis == 0:
        same = (ki // grid_w) == ((kj + shift) // grid_w)
    else:
        same = (ki % grid_w) == ((kj + shift) % grid_w)
    return (i < j) | ((ki >= 0) & (kj >= 0) & ~same)


def attention_mask(cfg: AxialConfig, layer, S, quirks: Quirks):
    """Additive [S,S] mask of one layer: oracle.dalle_local.attention_mask for global and local layers; for an axial
    layer the mask value where the query may not see the key (axial_hidden)."""
    if not cfg.is_axial(layer):
        return OL.attention_mask(cfg, layer, S, quirks)
    hidden = axial_hidden(S, cfg.text_seq_len, cfg.grid_w, AXES[cfg.attention_types[layer]])
    return hidden.to(torch.float32) * quirks.mask_value


def dropout_masks(dropout, B, cfg: AxialConfig):
    """oracle.dalle_local.dropout_masks without the attention-weight masks of axial layers either."""
    dm = OL.dropout_masks(dropout, B, cfg)
    dm["attn"] = [None if cfg.is_axial(l) else m for l, m in enumerate(dm["attn"])]
    return dm


def forward(params, tokens, cfg: AxialConfig, dropout=None, bf16=False, quirks: Quirks = None):
    """oracle.dalle_local.forward with axial layers: returns (loss, loss_batch, logits).  dropout: None (mode "eval")
    or (rates, seed, step, row0)."""
    q_ = quirks or Quirks()
    B, S = tokens.shape
    H, dh = cfg.n_heads, cfg.head_dim
    W = (lambda n: _r(params[n], bf16))
    none = [None] * cfg.n_layers
    dm = dropout_masks(dropout, B, cfg) if dropout is not None else \
        {"wte": None, "wpe": None, "attn": none, "attn_out": none, "mlp_out": none}
    drop = (lambda t, m: t if m is None else t * m)
    x = _r(drop(W("embedding/wte")[tokens], dm["wte"]) + drop(W("positional_embedding/wpe")[:S], dm["wpe"]), bf16)
    for l in range(cfg.n_layers):
        pre = f"layer_{l}/"
        mask = attention_mask(cfg, l, S, q_)
        h = _r(layer_norm(x, W(pre + "norm_1/g"), W(pre + "norm_1/b"), q_.ln_eps), bf16)
        q = _r(h @ W(pre + "attn/q"), bf16).view(B, S, H, dh)
        k = _r(h @ W(pre + "attn/k"), bf16).view(B, S, H, dh)
        v = _r(h @ W(pre + "attn/v"), bf16).view(B, S, H, dh)
        logits = torch.einsum("bihe,bjhe->bhij", q, k) * q_.attn_scale + mask
        p = _r(drop(torch.softmax(logits, dim=-1), dm["attn"][l]), bf16)
        a = _r(torch.einsum("bhij,bjhe->bihe", p, v).reshape(B, S, H * dh), bf16)
        a = _r(a @ W(pre + "attn/o") + W(pre + "attn/compute_output_bias/o_b"), bf16)
        if dm["attn_out"][l] is not None:
            a = _r(a * dm["attn_out"][l], bf16)
        x = _r(x + a, bf16)
        h = _r(layer_norm(x, W(pre + "norm_2/g"), W(pre + "norm_2/b"), q_.ln_eps), bf16)
        h1 = _r(torch.relu(h @ W(pre + "mlp/mlp_linear_1/kernel") + W(pre + "mlp/mlp_linear_1/bias")), bf16)
        h2 = _r(h1 @ W(pre + "mlp/mlp_linear_2/kernel") + W(pre + "mlp/mlp_linear_2/bias"), bf16)
        if dm["mlp_out"][l] is not None:
            h2 = _r(h2 * dm["mlp_out"][l], bf16)
        x = _r(x + h2, bf16)
    hf = _r(layer_norm(x, W("to_logits/layer_norm/g"), W("to_logits/layer_norm/b"), q_.ln_eps), bf16)
    logits = hf @ W("to_logits/linear_out/kernel") + W("to_logits/linear_out/bias")
    logits = logits.to(torch.promote_types(logits.dtype, torch.float32))
    labels = shift_labels(tokens, cfg.eos_token_id)
    loss_batch = torch.logsumexp(logits, -1) - logits.gather(-1, labels[..., None]).squeeze(-1)
    return loss_batch.mean(), loss_batch, logits


def loss_and_grads(params, tokens, cfg, dropout=None, bf16=False, quirks=None):
    """Autograd of forward(): (loss, loss_batch, logits, grads)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, loss_batch, logits = forward(leaves, tokens, cfg, dropout, bf16=bf16, quirks=quirks)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads


def kernel_order(S, text_len, grid_w, axis):
    """Sequence position of each kernel-order row t < text_len + grid_w^2 (attn_fa.cu): t itself for a row layer and
    for text rows; column-major over the image grid for a column layer."""
    t = torch.arange(text_len + grid_w * grid_w)
    if axis == 0:
        return t
    u = t - text_len
    return torch.where(t < text_len, t, text_len + (u % grid_w) * grid_w + u // grid_w)


def key_blocks(S, text_len, grid_w, qb, rows=64):
    """Kernel-order key blocks the forward / dQ kernels visit for query block qb (attn_fa.cu fa_axial_key_blocks and
    fa_axial_next, restated for 64-row blocks): the text blocks, then the blocks from the one holding the segment start
    of the block's first image query to qb."""
    jt = -(-text_len // rows)
    t = max(qb * rows, text_len)
    seg = 0 if t < text_len else text_len + (t - text_len) // grid_w * grid_w
    js = seg // rows if t < (qb + 1) * rows else jt
    j, out = (js if jt == 0 else 0), []
    while j <= qb:
        out.append(j)
        j = js if (jt <= j + 1 < js) else j + 1
    return out


def segment_hidden(S, text_len, grid_w):
    """[S,S] bool of the kernel-order mask: True unless t_k <= t_q and (t_k < text_len or t_k, t_q lie in the same
    segment of grid_w image rows)."""
    i = torch.arange(S)[:, None]
    j = torch.arange(S)[None, :]
    seg = lambda t: torch.div(t - text_len, grid_w, rounding_mode="floor")
    return (j > i) | ((j >= text_len) & (seg(j) != seg(i)))
