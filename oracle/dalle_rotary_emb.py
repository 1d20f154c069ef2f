"""ORACLE (test infrastructure, NOT product code) — the DALL-E transformer with DALLE-pytorch's rotary embedding
(rotary_emb) in place of learned positions.

With dh the head dim, TL the text length and W the side of the image-token grid (S = TL + W^2), rot = dh // 3 and
nf = rot // 2, pair m < 3 nf covers dims (2m, 2m+1) of a head and is rotated by the angle a_m(p) of the token at
sequence position p (dims 6 nf .. dh-1 are unchanged):

    part A, m = j < nf:       a = t theta_j,  theta_j = 1 / 10000^(2j / rot);   t = p (text), 8192 (every image token)
    part B, m = nf + j:       a = t phi_j,    phi_j = pi linspace(1, 5, nf)[j]; t = -10 (text), y[row] (image)
    part C, m = 2 nf + j:     a = t phi_j;                                      t = -10 (text), y[column] (image)
    y = linspace(-1, 1, W);   x_2m' = x_2m c - x_2m+1 s,   x_2m+1' = x_2m+1 c + x_2m s

The frequencies and the angle t * freq are float32 as torch computes them (DALLE-pytorch / rotary-embedding-torch);
cos and sin of the float32 angle are evaluated in float64 and rounded once to fp32 (table()).  The rotation applies
to q, k AND v of every head of every attention layer, after their bf16 cast, and is rounded to bf16 again.  There is
no learned position embedding: the input is wte[id] alone (the wpe term of oracle/dalle_gelu.py is a zero table, and
its dropout site masks zeros).

forward() is oracle/dalle_rotary.py's forward (itself oracle/dalle_gelu.py's) with this rotation in place of GPT-NeoX's;
with an all-zero angle table it computes bit for bit what oracle/dalle_gelu.forward computes with a zero wpe
(tests/test_rotary_emb_cpu.py).  It also takes gMLP layers ("mlp" in cfg.attention_types: oracle/dalle_gmlp.py's
block, not rotated) and the token shift after both LayerNorms (shift_tokens: oracle/dalle_shift.py's shift); the
attention masks and dropout masks come from `layers` (tests/conv_oracle.py, tests/block_sparse_oracle.py).
Mutations, each of which a correct engine must fail: "no_v" (v unrotated), "rotate_half" (GPT-NeoX pairs
(x_j, x_{j+3nf}) instead of interleaved ones), "swap_axes" (the row and column parts exchanged) and "image_text_pos"
(an image token's part-A position TL + k, its index in the sequence, instead of 8192).
"""
import math

import torch

from . import dalle_gelu as OG
from . import dalle_gmlp as OGM
from . import dalle_shift as OS
from .dalle import Quirks, _r, layer_norm, shift_labels

MUTATIONS = ("no_v", "rotate_half", "swap_axes", "image_text_pos")


def angles(text_len, grid_w, dh, mutate=None):
    """float32 [S, 3 nf] angles of every position (part A, then B, then C), DALLE-pytorch's recipe."""
    if mutate is not None and mutate not in MUTATIONS:
        raise ValueError(f"mutation {mutate!r} is not one of {MUTATIONS}")
    rot = dh // 3
    nf = rot // 2
    theta = 1.0 / (10000 ** (torch.arange(0, rot, 2)[:nf].float() / rot))
    phi = torch.linspace(1.0, 10 / 2, nf) * math.pi
    y = torch.linspace(-1.0, 1.0, grid_w)
    n_img = grid_w * grid_w
    img_pos = torch.arange(text_len, text_len + n_img, dtype=torch.float32) if mutate == "image_text_pos" else \
        torch.full((n_img,), 8192.0)
    t_a = torch.cat([torch.arange(text_len, dtype=torch.float32), img_pos])
    r, c = y.repeat_interleave(grid_w), y.repeat(grid_w)
    if mutate == "swap_axes":
        r, c = c, r
    t_b = torch.cat([torch.full((text_len,), -10.0), r])
    t_c = torch.cat([torch.full((text_len,), -10.0), c])
    return torch.cat([t_a[:, None] * theta, t_b[:, None] * phi, t_c[:, None] * phi], dim=1)


def table(text_len, grid_w, dh, dtype=torch.float32, mutate=None):
    """(cos, sin) [S, 3 nf] of angles(), evaluated in float64 and rounded once to dtype."""
    a = angles(text_len, grid_w, dh, mutate).double()
    return torch.cos(a).to(dtype), torch.sin(a).to(dtype)


def rotate(x, cos, sin, interleaved=True):
    """x [B, S, H, dh] with its first 3 nf pairs rotated by cos / sin [S, 3 nf] (x's dtype, each product and sum a
    separate operation; differentiable).  interleaved False: GPT-NeoX's (x_j, x_{j+n}) pairs (the "rotate_half"
    mutant)."""
    n = cos.shape[-1]
    c, s = cos.to(x.dtype)[None, :, None, :], sin.to(x.dtype)[None, :, None, :]
    if interleaved:
        a, b = x[..., 0:2 * n:2], x[..., 1:2 * n:2]
        rot = torch.stack([a * c - b * s, b * c + a * s], dim=-1).flatten(-2)
    else:
        a, b = x[..., :n], x[..., n:2 * n]
        rot = torch.cat([a * c - b * s, b * c + a * s], dim=-1)
    return torch.cat([rot, x[..., 2 * n:]], dim=-1)


def forward(params, tokens, cfg, dropout=None, bf16=False, quirks: Quirks = None, activation="relu", mutate=None,
            layers=None, rotary_mutate=None, tables=None, shift_tokens=False):
    """(loss, loss_batch, logits) of the rotary_emb model.  params has no positional_embedding/wpe.  tables: the
    (cos, sin) [S, 3 nf] to use instead of table() (the CPU tests' zero-angle check).  shift_tokens: DALLE-pytorch's
    token shift after both LayerNorms of every layer."""
    OG.check(activation, mutate)
    cfg, layers = OG._layers(cfg, layers)
    q_ = quirks or Quirks()
    B, S = tokens.shape
    H, dh = cfg.n_heads, cfg.head_dim
    W_ = math.isqrt(cfg.image_seq_len)
    dt = torch.float64 if not bf16 and params["embedding/wte"].dtype == torch.float64 else torch.float32
    cos, sin = tables if tables is not None else table(cfg.text_seq_len, W_, dh, dt, rotary_mutate)
    cos, sin = cos[:S], sin[:S]
    W = (lambda n: _r(params[n], bf16))
    none = [None] * cfg.n_layers
    dm = layers.dropout_masks(dropout, B, cfg) if dropout is not None else \
        {"wte": None, "wpe": None, "attn": none, "attn_out": none, "mlp_out": none}
    drop = (lambda t, m: t if m is None else t * m)
    il = rotary_mutate != "rotate_half"
    rot = (lambda t: _r(rotate(t, cos, sin, il), bf16))
    sh = (lambda t: OS.shift(t, cfg.text_seq_len, W_)) if shift_tokens else (lambda t: t)
    wte = W("embedding/wte")
    zero_pos = torch.zeros(S, wte.shape[1], dtype=wte.dtype)
    x = _r(drop(wte[tokens], dm["wte"]) + drop(zero_pos, dm["wpe"]), bf16)
    for l in range(cfg.n_layers):
        pre = f"layer_{l}/"
        h = sh(_r(layer_norm(x, W(pre + "norm_1/g"), W(pre + "norm_1/b"), q_.ln_eps), bf16))
        if OGM.is_mlp(cfg, l):   # a gMLP layer: not rotated
            a = OGM.gmlp_branch(h, params, pre, q_.ln_eps, bf16)
        else:
            mask = layers.attention_mask(cfg, l, S, q_)
            q = rot(_r(h @ W(pre + "attn/q"), bf16).view(B, S, H, dh))
            k = rot(_r(h @ W(pre + "attn/k"), bf16).view(B, S, H, dh))
            v = _r(h @ W(pre + "attn/v"), bf16).view(B, S, H, dh)
            if rotary_mutate != "no_v":
                v = rot(v)
            logits = torch.einsum("bihe,bjhe->bhij", q, k) * q_.attn_scale + mask
            p = _r(drop(torch.softmax(logits, dim=-1), dm["attn"][l]), bf16)
            a = _r(torch.einsum("bhij,bjhe->bihe", p, v).reshape(B, S, H * dh), bf16)
            a = _r(a @ W(pre + "attn/o") + W(pre + "attn/compute_output_bias/o_b"), bf16)
        if dm["attn_out"][l] is not None:
            a = _r(a * dm["attn_out"][l], bf16)
        x = _r(x + a, bf16)
        h = sh(_r(layer_norm(x, W(pre + "norm_2/g"), W(pre + "norm_2/b"), q_.ln_eps), bf16))
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
                   layers=None, rotary_mutate=None, shift_tokens=False):
    """Autograd of forward(): (loss, loss_batch, logits, grads)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, loss_batch, logits = forward(leaves, tokens, cfg, dropout, bf16=bf16, quirks=quirks, activation=activation,
                                       mutate=mutate, layers=layers, rotary_mutate=rotary_mutate,
                                       shift_tokens=shift_tokens)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads
