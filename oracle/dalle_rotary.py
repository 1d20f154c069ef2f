"""ORACLE (test infrastructure, NOT product code) — the DALL-E transformer with rotary position embeddings on q and k.

Rotary embeddings are not part of the reference; this is GPT-NeoX's definition (transformers' GPTNeoX
apply_rotary_pos_emb with partial_rotary_factor = r / head_dim, "rotate_half" layout), as DalleEngine(rotary_dim=r)
applies it:

    h = r / 2,  theta_j = base^(-2j / r),  c = cos(p theta_j),  s = sin(p theta_j)   (j < h, p the sequence index)
    x_j' = x_j c - x_{j+h} s,   x_{j+h}' = x_{j+h} c + x_j s,   dims r .. dh-1 unchanged

on q and k of every head of every layer, after their bf16 cast: q' = bf16(rot(q)), k' = bf16(rot(k)); v is unchanged.
cos and sin are evaluated in float64 and rounded once to fp32 (table()).

forward() is oracle/dalle_gelu.py's forward with that rotation inserted; rotary None or (0, base) rotates nothing and
then computes bit for bit what oracle/dalle_gelu.forward computes (tests/test_rotary_cpu.py).  Mutations, each of which
a correct engine must fail: "neg_theta" (rotation by -p theta_j), "interleaved" (GPT-J's pairs (x_2j, x_2j+1) instead
of rotate_half) and "shift" (the keys at positions p + 1, the queries at p: the off-by-one a decoder makes when it
rotates a step's key for the next position.  Shifting every position alike is no mutant: the scores depend on i - j
only).
"""
import torch

from . import dalle_gelu as OG
from .dalle import Quirks, _r, layer_norm, shift_labels

MUTATIONS = ("neg_theta", "interleaved", "shift")


def table(n_pos, r, base=10000.0, dtype=torch.float32):
    """(cos, sin) [n_pos, r / 2] of p theta_j, each evaluated in float64 and rounded once to dtype."""
    h = r // 2
    theta = torch.tensor([base ** (-2.0 * j / r) for j in range(h)], dtype=torch.float64)
    angle = torch.arange(n_pos, dtype=torch.float64)[:, None] * theta[None, :]
    return torch.cos(angle).to(dtype), torch.sin(angle).to(dtype)


def rotate(x, r, base=10000.0, mutate=None, positions=None):
    """x [B, S, H, dh] rotated over its first r dims at positions 0 .. S-1 (or `positions` [S]), in x's dtype, each
    product and sum a separate operation (differentiable)."""
    if mutate is not None and mutate not in MUTATIONS:
        raise ValueError(f"mutation {mutate!r} is not one of {MUTATIONS}")
    if not r:
        return x
    S, h = x.shape[1], r // 2
    pos = torch.arange(S) if positions is None else positions
    if mutate == "shift":
        pos = pos + 1
    c, s = table(int(pos.max()) + 1, r, base, torch.float32 if x.dtype != torch.float64 else torch.float64)
    c, s = c[pos].to(x.dtype)[None, :, None, :], s[pos].to(x.dtype)[None, :, None, :]
    if mutate == "neg_theta":
        s = -s
    if mutate == "interleaved":
        a, b = x[..., 0:r:2], x[..., 1:r:2]
        rot = torch.stack([a * c - b * s, b * c + a * s], dim=-1).flatten(-2)
    else:
        a, b = x[..., :h], x[..., h:r]
        rot = torch.cat([a * c - b * s, b * c + a * s], dim=-1)
    return torch.cat([rot, x[..., r:]], dim=-1)


def forward(params, tokens, cfg, dropout=None, bf16=False, quirks: Quirks = None, activation="relu", mutate=None,
            layers=None, rotary=None, rotary_mutate=None):
    """oracle/dalle_gelu.forward with q and k rotated: rotary = (r, base) (None: no rotation).  Returns (loss,
    loss_batch, logits)."""
    OG.check(activation, mutate)
    cfg, layers = OG._layers(cfg, layers)
    r, base = rotary if rotary is not None else (0, 10000.0)
    q_ = quirks or Quirks()
    B, S = tokens.shape
    H, dh = cfg.n_heads, cfg.head_dim
    W = (lambda n: _r(params[n], bf16))
    none = [None] * cfg.n_layers
    dm = layers.dropout_masks(dropout, B, cfg) if dropout is not None else \
        {"wte": None, "wpe": None, "attn": none, "attn_out": none, "mlp_out": none}
    drop = (lambda t, m: t if m is None else t * m)
    rot_q = (lambda t: _r(rotate(t, r, base, None if rotary_mutate == "shift" else rotary_mutate), bf16))
    rot_k = (lambda t: _r(rotate(t, r, base, rotary_mutate), bf16))
    x = _r(drop(W("embedding/wte")[tokens], dm["wte"]) + drop(W("positional_embedding/wpe")[:S], dm["wpe"]), bf16)
    for l in range(cfg.n_layers):
        pre = f"layer_{l}/"
        mask = layers.attention_mask(cfg, l, S, q_)
        h = _r(layer_norm(x, W(pre + "norm_1/g"), W(pre + "norm_1/b"), q_.ln_eps), bf16)
        q = rot_q(_r(h @ W(pre + "attn/q"), bf16).view(B, S, H, dh))
        k = rot_k(_r(h @ W(pre + "attn/k"), bf16).view(B, S, H, dh))
        v = _r(h @ W(pre + "attn/v"), bf16).view(B, S, H, dh)
        logits = torch.einsum("bihe,bjhe->bhij", q, k) * q_.attn_scale + mask
        p = _r(drop(torch.softmax(logits, dim=-1), dm["attn"][l]), bf16)
        a = _r(torch.einsum("bhij,bjhe->bihe", p, v).reshape(B, S, H * dh), bf16)
        a = _r(a @ W(pre + "attn/o") + W(pre + "attn/compute_output_bias/o_b"), bf16)
        if dm["attn_out"][l] is not None:
            a = _r(a * dm["attn_out"][l], bf16)
        x = _r(x + a, bf16)
        h = _r(layer_norm(x, W(pre + "norm_2/g"), W(pre + "norm_2/b"), q_.ln_eps), bf16)
        y = h @ W(pre + "mlp/mlp_linear_1/kernel") + W(pre + "mlp/mlp_linear_1/bias")
        h1 = _r(OG.mlp_activation(y, activation, bf16, mutate), bf16)
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


def loss_and_grads(params, tokens, cfg, dropout=None, bf16=False, quirks=None, activation="relu", mutate=None,
                   layers=None, rotary=None, rotary_mutate=None):
    """Autograd of forward(): (loss, loss_batch, logits, grads)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, loss_batch, logits = forward(leaves, tokens, cfg, dropout, bf16=bf16, quirks=quirks, activation=activation,
                                       mutate=mutate, layers=layers, rotary=rotary, rotary_mutate=rotary_mutate)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads
