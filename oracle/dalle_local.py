"""ORACLE (test infrastructure, NOT product code) — the reference DALL-E transformer with per-layer attention types.

The reference's DALLE.attention has two attention types (src/dalle_mtf/models.py:229-301): "global", the causal
attention oracle/dalle.py restates, and "local", mtf_transformer.attention.local_attention_1d with
fully_autoregressive=True and radius local_attention_radius (default 256, :259; incremental branch :257-273).
DALLE.block never passes attention_type (:326-335), so no reference config reaches the local branch; this module
restates the forward of oracle/dalle.py (and, with dropout, of oracle/dalle_dropout.py) with one type per layer.

Semantics (‡ recalled mtf 0.1.18 behaviour, like the ‡ items of oracle/dalle.py): in a local layer query i attends to
key j iff i - r < j <= i ("memory positions in the range (p - radius, p]").  mtf's block length (the largest divisor of
S <= max(r, 128)) does not change which keys are visible, and the zero-padded halo of the first block is masked through
sequence_id, so no query sees a pad key.  r >= S is causal attention.  A local layer gets no attention dropout: the
reference calls local_attention_1d(..., attention_kwargs={}) (:270); its residual dropout applies as in global layers
and the dropout site numbers do not move (site 2 + 3l is unused when layer l is local).

With every layer global, forward() computes operation for operation what oracle.dalle.forward (no dropout) and
oracle.dalle_dropout.forward (with dropout) compute (tests/test_local_attention_cpu.py).
"""
from dataclasses import dataclass

import torch

from . import dalle_dropout as D
from .dalle import DalleConfig, Quirks, _r, layer_norm, shift_labels


@dataclass
class LocalConfig(DalleConfig):
    attention_types: tuple = None      # one "global" | "local" per layer; None: every layer global
    local_attention_radius: int = 256  # src/dalle_mtf/models.py:259

    def is_local(self, layer):
        return self.attention_types is not None and self.attention_types[layer] == "local"


def attention_mask(cfg: LocalConfig, layer, S, quirks: Quirks):
    """Additive [S,S] mask of one layer: the mask value where query i may not see key j.  Global (models.py:221-227):
    j > i.  Local (models.py:257-273): also j <= i - radius."""
    i = torch.arange(S)[:, None]
    j = torch.arange(S)[None, :]
    hidden = i < j
    if cfg.is_local(layer):
        hidden = hidden | (j <= i - cfg.local_attention_radius)
    return hidden.to(torch.float32) * quirks.mask_value


def dropout_masks(dropout, B, cfg: LocalConfig):
    """oracle.dalle_dropout.dropout_masks without the attention-weight masks of local layers."""
    dm = D.dropout_masks(dropout, B, cfg)
    dm["attn"] = [None if cfg.is_local(l) else m for l, m in enumerate(dm["attn"])]
    return dm


def forward(params, tokens, cfg: LocalConfig, dropout=None, bf16=False, quirks: Quirks = None):
    """DALLE.forward (src/dalle_mtf/models.py:397-416) with per-layer attention types: returns (loss, loss_batch,
    logits).  dropout: None (mode "eval") or (rates, seed, step, row0) as oracle.dalle_dropout.forward takes it."""
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
        logits = torch.einsum("bihe,bjhe->bhij", q, k) * q_.attn_scale + mask              # fp32 ‡
        p = _r(drop(torch.softmax(logits, dim=-1), dm["attn"][l]), bf16)                   # :290-299
        a = _r(torch.einsum("bhij,bjhe->bihe", p, v).reshape(B, S, H * dh), bf16)
        a = _r(a @ W(pre + "attn/o") + W(pre + "attn/compute_output_bias/o_b"), bf16)      # :303-311
        if dm["attn_out"][l] is not None:
            a = _r(a * dm["attn_out"][l], bf16)                                             # :312-314
        x = _r(x + a, bf16)                                                                 # :330
        h = _r(layer_norm(x, W(pre + "norm_2/g"), W(pre + "norm_2/b"), q_.ln_eps), bf16)
        h1 = _r(torch.relu(h @ W(pre + "mlp/mlp_linear_1/kernel") + W(pre + "mlp/mlp_linear_1/bias")), bf16)
        h2 = _r(h1 @ W(pre + "mlp/mlp_linear_2/kernel") + W(pre + "mlp/mlp_linear_2/bias"), bf16)
        if dm["mlp_out"][l] is not None:
            h2 = _r(h2 * dm["mlp_out"][l], bf16)                                           # :321-323
        x = _r(x + h2, bf16)                                                                # :333
    hf = _r(layer_norm(x, W("to_logits/layer_norm/g"), W("to_logits/layer_norm/b"), q_.ln_eps), bf16)
    logits = hf @ W("to_logits/linear_out/kernel") + W("to_logits/linear_out/bias")
    logits = logits.to(torch.promote_types(logits.dtype, torch.float32))                   # :395
    labels = shift_labels(tokens, cfg.eos_token_id)
    loss_batch = torch.logsumexp(logits, -1) - logits.gather(-1, labels[..., None]).squeeze(-1)
    return loss_batch.mean(), loss_batch, logits


def loss_and_grads(params, tokens, cfg, dropout=None, bf16=False, quirks=None):
    """Autograd of forward() (mtf.gradients, src/optimizers.py:34): (loss, loss_batch, logits, grads)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, loss_batch, logits = forward(leaves, tokens, cfg, dropout, bf16=bf16, quirks=quirks)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads
