"""ORACLE (test infrastructure, NOT product code) — the reference DALL-E transformer in mode "train" with dropout.

oracle/dalle.py restates the reference without dropout (every reference config leaves the rates at 0).  This module
restates the same forward (oracle.dalle.forward, faithful=False) with mtf.dropout applied where the reference applies
it when a rate is above 0 (src/dalle_mtf/models.py:198-200, 215-217, 290-299, 312-314, 321-323), under the masks of
oracle/philox.py.  The reference draws its masks from the TPU's stateful RNG, which cannot be reproduced, so parity
means the reference's math under these masks.  Two semantics are recalled mtf 0.1.18 behaviour (‡): mtf.dropout draws
i.i.d. masks over the tensor's full shape and scales kept values by 1 / (1 - rate), and attention dropout acts on the
normalised weights before the PV product.

dropout = (rates, seed, step, row0): rates = (embed, attention, residual), row0 = global index of tokens[0].
With every rate 0 the computation is oracle.dalle.forward's, operation for operation (tests/test_dropout_cpu.py).
"""
import torch

from . import philox as X
from .dalle import DalleConfig, Quirks, _r, layer_norm, shift_labels


def dropout_masks(dropout, B, cfg: DalleConfig):
    """keep * scale multipliers (fp32) of every site, None where the rate is 0: wte [B, S, d], wpe [S, d] (one mask for
    the whole batch: models.py:215-217 drops pos_emb before it is broadcast over the batch), attention [B, H, S, S]
    per layer, attention output and MLP output [B, S, d] per layer."""
    (emb, att, res), seed, step, row0 = dropout
    S, d, H, L = cfg.seq_len, cfg.n_embd, cfg.n_heads, cfg.n_layers

    def elem(rate, site, rows, r0):
        if not rate:
            return None
        keep = X.keep_elementwise(rate, seed, step, site, rows, d, r0)
        return torch.from_numpy(keep).float() * X.threshold_scale(rate)[1]

    def tokens(rate, site):
        m = elem(rate, site, B * S, row0 * S)
        return None if m is None else m.view(B, S, d)

    def attn(site):
        if not att:
            return None
        return torch.from_numpy(X.keep_attention(att, seed, step, site, B, H, S, row0)).float() * \
            X.threshold_scale(att)[1]

    return {
        "wte": tokens(emb, X.SITE_WTE), "wpe": elem(emb, X.SITE_WPE, S, 0),
        "attn": [attn(X.site_attn(l)) for l in range(L)],
        "attn_out": [tokens(res, X.site_attn_out(l)) for l in range(L)],
        "mlp_out": [tokens(res, X.site_mlp_out(l)) for l in range(L)],
    }


def forward(params, tokens, cfg: DalleConfig, dropout, bf16=False, quirks: Quirks = None):
    """oracle.dalle.forward in mode "train": returns (loss, loss_batch, logits)."""
    q_ = quirks or Quirks()
    B, S = tokens.shape
    H, dh = cfg.n_heads, cfg.head_dim
    W = (lambda n: _r(params[n], bf16))
    dm = dropout_masks(dropout, B, cfg)
    drop = (lambda t, m: t if m is None else t * m)
    # embedding (models.py:186-201) + positional embedding (models.py:203-219), each dropped
    x = _r(drop(W("embedding/wte")[tokens], dm["wte"]) + drop(W("positional_embedding/wpe")[:S], dm["wpe"]), bf16)
    i = torch.arange(S)[:, None]
    j = torch.arange(S)[None, :]
    mask = (i < j).to(torch.float32) * q_.mask_value
    for l in range(cfg.n_layers):
        pre = f"layer_{l}/"
        h = _r(layer_norm(x, W(pre + "norm_1/g"), W(pre + "norm_1/b"), q_.ln_eps), bf16)
        q = _r(h @ W(pre + "attn/q"), bf16).view(B, S, H, dh)
        k = _r(h @ W(pre + "attn/k"), bf16).view(B, S, H, dh)
        v = _r(h @ W(pre + "attn/v"), bf16).view(B, S, H, dh)
        logits = torch.einsum("bihe,bjhe->bhij", q, k) * q_.attn_scale + mask
        p = _r(drop(torch.softmax(logits, dim=-1), dm["attn"][l]), bf16)               # ‡ :290-299
        a = _r(torch.einsum("bhij,bjhe->bihe", p, v).reshape(B, S, H * dh), bf16)
        a = _r(a @ W(pre + "attn/o") + W(pre + "attn/compute_output_bias/o_b"), bf16)
        if dm["attn_out"][l] is not None:
            a = _r(a * dm["attn_out"][l], bf16)                                          # :312-314
        x = _r(x + a, bf16)
        h = _r(layer_norm(x, W(pre + "norm_2/g"), W(pre + "norm_2/b"), q_.ln_eps), bf16)
        h1 = _r(torch.relu(h @ W(pre + "mlp/mlp_linear_1/kernel") + W(pre + "mlp/mlp_linear_1/bias")), bf16)
        h2 = _r(h1 @ W(pre + "mlp/mlp_linear_2/kernel") + W(pre + "mlp/mlp_linear_2/bias"), bf16)
        if dm["mlp_out"][l] is not None:
            h2 = _r(h2 * dm["mlp_out"][l], bf16)                                        # :321-323
        x = _r(x + h2, bf16)
    hf = _r(layer_norm(x, W("to_logits/layer_norm/g"), W("to_logits/layer_norm/b"), q_.ln_eps), bf16)
    logits = hf @ W("to_logits/linear_out/kernel") + W("to_logits/linear_out/bias")
    logits = logits.to(torch.promote_types(logits.dtype, torch.float32))
    labels = shift_labels(tokens, cfg.eos_token_id)
    loss_batch = torch.logsumexp(logits, -1) - logits.gather(-1, labels[..., None]).squeeze(-1)
    return loss_batch.mean(), loss_batch, logits


def loss_and_grads(params, tokens, cfg, dropout, bf16=False, quirks=None):
    """Autograd of forward() (mtf.gradients, src/optimizers.py:34): (loss, loss_batch, logits, grads)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, loss_batch, logits = forward(leaves, tokens, cfg, dropout, bf16=bf16, quirks=quirks)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads
