"""ORACLE (test infrastructure, NOT product code) — the DALL-E transformer with DALLE-pytorch's token shift.

DALLE-pytorch wraps every attention and feed-forward block as PreNorm(dim, PreShiftToken(block)): the block reads the
LayerNorm output with part of its features taken from earlier tokens.  This engine's sequence (DALLE-mtf's) has no
<bos>: positions p < TL = text_seq_len are text, the rest the image tokens of a W x W grid (image_seq_len = W^2).
With c = d / 4 and y a LayerNorm output [..., S, d], shift(y) keeps y[p, 2c:d) and takes

    text p          : y[p-1, 0:2c)                                 (zeros at p = 0)
    image (r, k)    : y[p-W, 0:c) if r >= 1 ("top"),  y[p-1, c:2c) if k >= 1 ("left"),  zeros otherwise

Text never reads image rows and image never reads text rows, the rule DALLE-pytorch applies to its text part (shift
of chunk(2)[0] by one position) and its image part (chunk(4)[0] from the top, chunk(4)[1] from the left, zero
padded).  The shift moves bf16 values and rounds nothing.

forward() is oracle/dalle_glu.forward (activation, gated, rotary, the attention layers from `layers`) with the shift
applied after both LayerNorms of every layer; shift=False computes bit for bit what that forward computes
(tests/test_shift_tokens_cpu.py).  Mutations a correct engine must fail:
  * "swap":     the top and left sources exchanged;
  * "flat":     a 1-D shift by one position of [0, 2c) over the whole sequence (no grid, no text / image boundary);
  * "pre_norm": the shift applied to x before the LayerNorm instead of to its output.
"""
import math

import torch

from . import dalle_gelu as OG
from . import dalle_glu as OGL
from .dalle import Quirks, _r, layer_norm, shift_labels
from .dalle_rotary import rotate

MUTATIONS = ("swap", "flat", "pre_norm")


def sources(S, text_len, grid_w, mutate=None):
    """(top, left) int64 [S]: the position chunk [0, c) and chunk [c, 2c) of each position read, -1 for zeros."""
    top, left = [], []
    for p in range(S):
        if mutate == "flat" or p < text_len:
            t = le = p - 1
        else:
            u = p - text_len
            t = p - grid_w if u >= grid_w else -1
            le = p - 1 if u % grid_w else -1
        if mutate == "swap":
            t, le = le, t
        top.append(t)
        left.append(le)
    return torch.tensor(top), torch.tensor(left)


def shift(y, text_len, grid_w, mutate=None):
    """shift(y) of y [..., S, d] (differentiable: a gather from y with a zero row in front)."""
    S, d = y.shape[-2], y.shape[-1]
    c = d // 4
    top, left = sources(S, text_len, grid_w, mutate)
    yp = torch.cat([torch.zeros_like(y[..., :1, :]), y], -2)
    return torch.cat([yp[..., top + 1, :c], yp[..., left + 1, c:2 * c], y[..., 2 * c:]], -1)


def check(mutate):
    if mutate is not None and mutate not in MUTATIONS:
        raise ValueError(f"mutation {mutate!r} is not one of {MUTATIONS}")


def forward(params, tokens, cfg, dropout=None, bf16=False, quirks: Quirks = None, activation="relu", gated=False,
            mutate=None, layers=None, rotary=None, shift_tokens=True, shift_mutate=None):
    """DALLE.forward (src/dalle_mtf/models.py:397-416) with the token shift after both LayerNorms (shift_tokens=False:
    oracle/dalle_glu.forward with the same arguments, bit for bit): returns (loss, loss_batch, logits).  mutate is the
    gated MLP's mutation (oracle/dalle_glu.py), shift_mutate the shift's.  dropout: None or (rates, seed, step, row0)."""
    OGL.check(activation, mutate)
    check(shift_mutate)
    if shift_mutate is not None and not shift_tokens:
        raise ValueError("the mutations are of the token shift")
    if mutate is not None and not gated:
        raise ValueError("the mutations are of the gated MLP")
    cfg, layers = OG._layers(cfg, layers)
    q_ = quirks or Quirks()
    B, S = tokens.shape
    H, dh = cfg.n_heads, cfg.head_dim
    TL, Wg = cfg.text_seq_len, math.isqrt(cfg.image_seq_len)
    W = (lambda n: _r(params[n], bf16))
    none = [None] * cfg.n_layers
    dm = layers.dropout_masks(dropout, B, cfg) if dropout is not None else \
        {"wte": None, "wpe": None, "attn": none, "attn_out": none, "mlp_out": none}
    drop = (lambda t, m: t if m is None else t * m)
    rot = (lambda t: t) if rotary is None else (lambda t: _r(rotate(t, rotary[0], rotary[1]), bf16))
    sh = (lambda t: t) if not shift_tokens else (lambda t: shift(t, TL, Wg, shift_mutate))
    pre, post = (sh, lambda t: t) if shift_mutate == "pre_norm" else (lambda t: t, sh)

    def norm(x, name):
        return post(_r(layer_norm(pre(x), W(name + "/g"), W(name + "/b"), q_.ln_eps), bf16))

    x = _r(drop(W("embedding/wte")[tokens], dm["wte"]) + drop(W("positional_embedding/wpe")[:S], dm["wpe"]), bf16)
    for l in range(cfg.n_layers):
        pfx = f"layer_{l}/"
        mask = layers.attention_mask(cfg, l, S, q_)
        h = norm(x, pfx + "norm_1")
        q = rot(_r(h @ W(pfx + "attn/q"), bf16).view(B, S, H, dh))
        k = rot(_r(h @ W(pfx + "attn/k"), bf16).view(B, S, H, dh))
        v = _r(h @ W(pfx + "attn/v"), bf16).view(B, S, H, dh)
        logits = torch.einsum("bihe,bjhe->bhij", q, k) * q_.attn_scale + mask              # fp32 ‡
        p = _r(drop(torch.softmax(logits, dim=-1), dm["attn"][l]), bf16)
        a = _r(torch.einsum("bhij,bjhe->bihe", p, v).reshape(B, S, H * dh), bf16)
        a = _r(a @ W(pfx + "attn/o") + W(pfx + "attn/compute_output_bias/o_b"), bf16)
        if dm["attn_out"][l] is not None:
            a = _r(a * dm["attn_out"][l], bf16)
        x = _r(x + a, bf16)
        h = norm(x, pfx + "norm_2")
        y = h @ W(pfx + "mlp/mlp_linear_1/kernel") + W(pfx + "mlp/mlp_linear_1/bias")
        if gated:
            h1 = OGL.gated_mlp(y, activation, bf16, mutate)
        else:
            h1 = _r(OG.mlp_activation(y, activation, bf16), bf16)
        h2 = _r(h1 @ W(pfx + "mlp/mlp_linear_2/kernel") + W(pfx + "mlp/mlp_linear_2/bias"), bf16)
        if dm["mlp_out"][l] is not None:
            h2 = _r(h2 * dm["mlp_out"][l], bf16)
        x = _r(x + h2, bf16)
    hf = _r(layer_norm(x, W("to_logits/layer_norm/g"), W("to_logits/layer_norm/b"), q_.ln_eps), bf16)
    logits = hf @ W("to_logits/linear_out/kernel") + W("to_logits/linear_out/bias")
    logits = logits.to(torch.promote_types(logits.dtype, torch.float32))
    labels = shift_labels(tokens, cfg.eos_token_id)
    loss_batch = torch.logsumexp(logits, -1) - logits.gather(-1, labels[..., None]).squeeze(-1)
    return loss_batch.mean(), loss_batch, logits


def loss_and_grads(params, tokens, cfg, dropout=None, bf16=False, quirks=None, activation="relu", gated=False,
                   mutate=None, layers=None, rotary=None, shift_tokens=True, shift_mutate=None):
    """Autograd of forward(): (loss, loss_batch, logits, grads)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, loss_batch, logits = forward(leaves, tokens, cfg, dropout, bf16=bf16, quirks=quirks, activation=activation,
                                       gated=gated, mutate=mutate, layers=layers, rotary=rotary,
                                       shift_tokens=shift_tokens, shift_mutate=shift_mutate)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads
