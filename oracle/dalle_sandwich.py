"""ORACLE (test infrastructure, NOT product code) — the DALL-E transformer with sandwich LayerNorm.

CogView's Sandwich-LN, as DALLE-pytorch builds it with PreNorm(dim, fn, sandwich=True) ‡: the output of each branch,
after the branch's own dropout, goes through a LayerNorm of its own before the residual add.  Layer l becomes

    a    = attn(LN1(x))                    unchanged (token shift, rotary, every attention type)
    oa   = bf16(drop_attn_out(a Wo + o_b))  the residual-dropout site "attn_out" of layer l, no residual
    xmid = bf16(x + LNa(oa))               LNa: layer_l/attn/norm_out/{g,b}
    h    = mlp(LN2(xmid))                  unchanged (ReLU, GELU, ReGLU / GEGLU)
    om   = bf16(drop_mlp_out(h W2 + b2))   site "mlp_out" of layer l, no residual
    xout = bf16(xmid + LNm(om))            LNm: layer_l/mlp/norm_out/{g,b}

Both norms use the model's ln_eps.  The normalised branch is never rounded on its own: x + (o - mean) rstd g + b is
rounded once.  (‡ DALLE-pytorch's placement of norm_out after the branch's dropout is recalled, not checked against
its source.)

forward() is oracle/dalle_shift.forward with the two norms added; sandwich_norm=False computes bit for bit what that
forward computes (tests/test_sandwich_norm_cpu.py).  Mutations a correct engine must fail:
  * "post_ln":          x = LN(x + o) with the branch's norm_out parameters (post-LN instead of the sandwich);
  * "norm_before_drop": x + drop(LN(o)), the residual dropout applied after the norm;
  * "swapped":          LNa's parameters used on the MLP branch and LNm's on the attention branch;
  * "ignored":          the new norms skipped (x + o).
"""
import math

import torch

from . import dalle_gelu as OG
from . import dalle_glu as OGL
from . import dalle_shift as OS
from .dalle import Quirks, _r, layer_norm, shift_labels
from .dalle_rotary import rotate

MUTATIONS = ("post_ln", "norm_before_drop", "swapped", "ignored")


def norm_names(n_layers):
    """The variables sandwich_norm adds, in layer order."""
    return [f"layer_{l}/{b}/norm_out/{v}" for l in range(n_layers) for b in ("attn", "mlp") for v in ("g", "b")]


def init_params(params, cfg, seed=None):
    """params plus the sandwich norms: g = 1, b = 0 (the engine's initialisation), or with a seed g ~ 1 + 0.3 N(0, 1)
    and b ~ 0.1 N(0, 1), so that a test can tell the two norms apart."""
    out = dict(params)
    g = torch.Generator().manual_seed(seed) if seed is not None else None
    d = cfg.n_embd
    for name in norm_names(cfg.n_layers):
        if g is None:
            out[name] = torch.ones(d) if name.endswith("/g") else torch.zeros(d)
        elif name.endswith("/g"):
            out[name] = 1 + torch.randn(d, generator=g) * 0.3
        else:
            out[name] = torch.randn(d, generator=g) * 0.1
    return out


def check(mutate):
    if mutate is not None and mutate not in MUTATIONS:
        raise ValueError(f"mutation {mutate!r} is not one of {MUTATIONS}")


def forward(params, tokens, cfg, dropout=None, bf16=False, quirks: Quirks = None, activation="relu", gated=False,
            mutate=None, layers=None, rotary=None, shift_tokens=False, shift_mutate=None, sandwich_norm=True,
            sandwich_mutate=None):
    """DALLE.forward (src/dalle_mtf/models.py:397-416) with the sandwich LayerNorm (sandwich_norm=False:
    oracle/dalle_shift.forward with the same arguments, bit for bit): returns (loss, loss_batch, logits).  mutate is the
    gated MLP's mutation, shift_mutate the token shift's, sandwich_mutate this oracle's.  dropout: None or
    (rates, seed, step, row0)."""
    check(sandwich_mutate)
    if sandwich_mutate is not None and not sandwich_norm:
        raise ValueError("the mutations are of the sandwich LayerNorm")
    OGL.check(activation, mutate)
    OS.check(shift_mutate)
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
    sh = (lambda t: t) if not shift_tokens else (lambda t: OS.shift(t, TL, Wg, shift_mutate))
    pre, post = (sh, lambda t: t) if shift_mutate == "pre_norm" else (lambda t: t, sh)

    def norm(x, name):
        return post(_r(layer_norm(pre(x), W(name + "/g"), W(name + "/b"), q_.ln_eps), bf16))

    def sandwich(x, o, mask, name):
        """x + LN_name(drop(o)) with o = the branch output before its dropout, one rounding (or a mutant of it);
        without the sandwich LayerNorm x + drop(o), as oracle/dalle_shift.forward rounds it."""
        ln = (lambda t: layer_norm(t, W(name + "/g"), W(name + "/b"), q_.ln_eps))
        if sandwich_mutate == "norm_before_drop":
            return _r(x + drop(ln(o), mask), bf16)
        if mask is not None:
            o = _r(o * mask, bf16)
        if not sandwich_norm or sandwich_mutate == "ignored":
            return _r(x + o, bf16)
        if sandwich_mutate == "post_ln":
            return _r(ln(_r(x + o, bf16)), bf16)
        return _r(x + ln(o), bf16)

    names = {"attn": "attn/norm_out", "mlp": "mlp/norm_out"}
    if sandwich_mutate == "swapped":
        names = {"attn": "mlp/norm_out", "mlp": "attn/norm_out"}
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
        x = sandwich(x, a, dm["attn_out"][l], pfx + names["attn"])
        h = norm(x, pfx + "norm_2")
        y = h @ W(pfx + "mlp/mlp_linear_1/kernel") + W(pfx + "mlp/mlp_linear_1/bias")
        if gated:
            h1 = OGL.gated_mlp(y, activation, bf16, mutate)
        else:
            h1 = _r(OG.mlp_activation(y, activation, bf16), bf16)
        h2 = _r(h1 @ W(pfx + "mlp/mlp_linear_2/kernel") + W(pfx + "mlp/mlp_linear_2/bias"), bf16)
        x = sandwich(x, h2, dm["mlp_out"][l], pfx + names["mlp"])
    hf = _r(layer_norm(x, W("to_logits/layer_norm/g"), W("to_logits/layer_norm/b"), q_.ln_eps), bf16)
    logits = hf @ W("to_logits/linear_out/kernel") + W("to_logits/linear_out/bias")
    logits = logits.to(torch.promote_types(logits.dtype, torch.float32))
    labels = shift_labels(tokens, cfg.eos_token_id)
    loss_batch = torch.logsumexp(logits, -1) - logits.gather(-1, labels[..., None]).squeeze(-1)
    return loss_batch.mean(), loss_batch, logits


def loss_and_grads(params, tokens, cfg, dropout=None, bf16=False, quirks=None, activation="relu", gated=False,
                   mutate=None, layers=None, rotary=None, shift_tokens=False, shift_mutate=None, sandwich_norm=True,
                   sandwich_mutate=None):
    """Autograd of forward(): (loss, loss_batch, logits, grads)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, loss_batch, logits = forward(leaves, tokens, cfg, dropout, bf16=bf16, quirks=quirks, activation=activation,
                                       gated=gated, mutate=mutate, layers=layers, rotary=rotary,
                                       shift_tokens=shift_tokens, shift_mutate=shift_mutate,
                                       sandwich_norm=sandwich_norm, sandwich_mutate=sandwich_mutate)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads
