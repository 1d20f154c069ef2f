"""Float64 / fp32 reference of DALL-E transformers with convolutional attention layers, for the tests.

Convolutional layers are an extension, not in the reference: DALL-E's convolutional mask, DALLE-pytorch's
SparseConvCausalAttention at dilation 1.  With TL = text_seq_len, the image tokens on a W x W grid
(image_seq_len = W^2) and kernel size k, text queries are causal, as in a global layer, and the image query at grid row
r, column c sees every text key plus the image keys (r', c') with r - k < r' <= r and c - k < c' <= c: the k x k window
above and to the left of it.  The mask is built here from (r, c).  Convolutional layers get no attention dropout (the
dropout site 2 + 3l of a conv layer l is unused) and keep their residual dropout.

Global, local and axial layers take tests/axial_oracle.py's masks, and forward() is axial_oracle.forward operation for
operation, so a model without conv layers computes bit for bit what that module computes.
"""
from dataclasses import dataclass

import torch

import axial_oracle as OA
from oracle.dalle import Quirks, _r, layer_norm, shift_labels


@dataclass
class ConvConfig(OA.AxialConfig):
    """axial_oracle.AxialConfig whose attention_types may also hold "conv", of kernel size conv_attention_kernel."""
    conv_attention_kernel: int = 5

    def is_conv(self, layer):
        return self.attention_types is not None and self.attention_types[layer] == "conv"


def conv_hidden(S, text_len, grid_w, kernel):
    """[S,S] bool: True where query i may not see key j in a convolutional layer of kernel size `kernel`."""
    i = torch.arange(S)[:, None]
    j = torch.arange(S)[None, :]
    ki, kj = i - text_len, j - text_len
    ri, ci = torch.div(ki, grid_w, rounding_mode="floor"), ki % grid_w
    rj, cj = torch.div(kj, grid_w, rounding_mode="floor"), kj % grid_w
    window = (rj > ri - kernel) & (rj <= ri) & (cj <= ci) & (cj > ci - kernel)
    return (j > i) | ((kj >= 0) & ~((ki >= 0) & window))


def attention_mask(cfg: ConvConfig, layer, S, quirks: Quirks):
    """Additive [S,S] mask of one layer: axial_oracle.attention_mask for global, local and axial layers; for a conv layer
    the mask value where the query may not see the key (conv_hidden)."""
    if not cfg.is_conv(layer):
        return OA.attention_mask(cfg, layer, S, quirks)
    hidden = conv_hidden(S, cfg.text_seq_len, cfg.grid_w, cfg.conv_attention_kernel)
    return hidden.to(torch.float32) * quirks.mask_value


def dropout_masks(dropout, B, cfg: ConvConfig):
    """axial_oracle.dropout_masks without the attention-weight masks of conv layers either."""
    dm = OA.dropout_masks(dropout, B, cfg)
    dm["attn"] = [None if cfg.is_conv(l) else m for l, m in enumerate(dm["attn"])]
    return dm


def forward(params, tokens, cfg: ConvConfig, dropout=None, bf16=False, quirks: Quirks = None):
    """axial_oracle.forward with conv layers: returns (loss, loss_batch, logits).  dropout: None (mode "eval") or
    (rates, seed, step, row0)."""
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


# ---- the kernels' tile walks (dalle_mtf_b200/csrc/attn_fa.cu, CONV), restated for 64-row blocks
def key_blocks(S, text_len, grid_w, kernel, qb, rows=64):
    """Key blocks the forward / dQ kernels visit for query block qb: the text blocks, then the band from the block
    holding the first position of the window's top row (of the block's first image query) to qb."""
    jt = -(-text_len // rows)
    t = max(qb * rows, text_len)
    top = max(0, (t - text_len) // grid_w - kernel + 1)
    js = (text_len + top * grid_w) // rows if t < (qb + 1) * rows else jt
    j, out = (js if jt == 0 else 0), []
    while j <= qb:
        out.append(j)
        j = js if (jt <= j + 1 < js) else j + 1
    return out


def query_blocks(S, text_len, grid_w, kernel, kb, rows=64):
    """Query blocks the dK / dV kernel visits for key block kb: every later one for a block holding a text key, else
    up to the block of position min(S - 1, last key + (min(k, W) - 1) (W + 1))."""
    nq, k0 = -(-S // rows), kb * rows
    if k0 < text_len:
        return list(range(kb, nq))
    last = min(k0 + rows - 1, S - 1)
    reach = last + (min(kernel, grid_w) - 1) * (grid_w + 1)
    return list(range(kb, min(nq, reach // rows + 1)))
