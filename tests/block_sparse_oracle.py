"""Float64 / fp32 reference of DALL-E transformers with block-sparse attention layers, for the tests.

Block-sparse layers are an extension, not in the reference: DALLE-pytorch's SparseAttention, a DeepSpeed
VariableSparsityConfig layout.  The layout is an input here: cfg.block_sparse_layouts[l] is the bool [nb, nb] block
layout of layer l (dalle_engine.block_sparse_layout draws it), of blocks of cfg.sparse_block_size tokens.  Query i
sees key j iff j <= i and layout[i // b][j // b].  Block-sparse layers get no attention dropout (the dropout site
2 + 3l of such a layer l is unused) and keep their residual dropout.

Global, local, axial and conv layers take tests/conv_oracle.py's masks, and forward() is conv_oracle.forward operation
for operation, so a model without block-sparse layers computes bit for bit what that module computes.
"""
from dataclasses import dataclass

import torch

import conv_oracle as OC
from oracle.dalle import Quirks, _r, layer_norm, shift_labels


@dataclass
class BlockSparseConfig(OC.ConvConfig):
    """conv_oracle.ConvConfig whose attention_types may also hold "block_sparse", with per-layer block layouts."""
    sparse_block_size: int = 16
    block_sparse_layouts: tuple = None

    def is_block_sparse(self, layer):
        return self.attention_types is not None and self.attention_types[layer] == "block_sparse"


def block_sparse_hidden(S, layout, block):
    """[S,S] bool: True where query i may not see key j under the block layout."""
    lay = torch.as_tensor(layout, dtype=torch.bool)
    g = torch.arange(S) // block
    i = torch.arange(S)[:, None]
    j = torch.arange(S)[None, :]
    return (j > i) | ~lay[g][:, g]


def attention_mask(cfg: BlockSparseConfig, layer, S, quirks: Quirks):
    """Additive [S,S] mask of one layer: conv_oracle.attention_mask for global, local, axial and conv layers; for a
    block-sparse layer the mask value where the query may not see the key (block_sparse_hidden)."""
    if not cfg.is_block_sparse(layer):
        return OC.attention_mask(cfg, layer, S, quirks)
    hidden = block_sparse_hidden(S, cfg.block_sparse_layouts[layer], cfg.sparse_block_size)
    return hidden.to(torch.float32) * quirks.mask_value


def dropout_masks(dropout, B, cfg: BlockSparseConfig):
    """conv_oracle.dropout_masks without the attention-weight masks of block-sparse layers either."""
    dm = OC.dropout_masks(dropout, B, cfg)
    dm["attn"] = [None if cfg.is_block_sparse(l) else m for l, m in enumerate(dm["attn"])]
    return dm


def forward(params, tokens, cfg: BlockSparseConfig, dropout=None, bf16=False, quirks: Quirks = None):
    """conv_oracle.forward with block-sparse layers: returns (loss, loss_batch, logits).  dropout: None (mode "eval")
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
