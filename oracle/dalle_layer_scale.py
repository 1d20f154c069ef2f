"""ORACLE (test infrastructure, NOT product code) — the DALL-E transformer with LayerScale and DALLE-pytorch's stable.

DALLE-pytorch wraps every branch of every layer in LayerScale(dim, depth, PreNorm(...)): the branch output is
multiplied per channel by a learned vector before the residual add.  Per layer l, with oa the token mixer's output
(attention or gMLP) after its residual dropout and om the MLP's:

    xmid = bf16(x    + s_a oa)          with the sandwich LayerNorm: bf16(x    + s_a LNa(oa)), one rounding
    xout = bf16(xmid + s_m om)          with the sandwich LayerNorm: bf16(xmid + s_m LNm(om))

s_a is layer_l/attn/layer_scale (layer_l/gmlp/layer_scale in an 'mlp' layer) and s_m layer_l/mlp/layer_scale, both
[d].  DALLE-pytorch initialises them by depth n = l + 1 (recalled, not checked): 0.1 for n <= 18, 1e-5 for
18 < n <= 24, 1e-6 beyond; a number instead of true starts every layer at that number.

stable (recalled, not checked): (1) the embedding's gradient shrinks, tokens * alpha + tokens.detach() * (1 - alpha)
with alpha = 0.1: the forward is the same, every embedding table's gradient is alpha times what it was; (2) DivideMax
before the final LayerNorm: per row m = max_c x[c] of the bf16 values, detached, u = x / m in fp32 (never rounded to
bf16), hf = bf16(LN_f(u)); (3) its stable softmax equals softmax, which this oracle computes in fp32 already.

forward() is oracle/dalle_gmlp.forward with both added; with layer_scale=False and stable=False it computes bit for bit
what that forward computes (tests/test_layer_scale_cpu.py).  Mutations a correct engine must fail:
  * "post_residual":     xmid = bf16((x + oa) s_a), the scale applied after the residual add;
  * "scale_before_norm": with the sandwich LayerNorm, x + LNa(s_a oa): the scale inside the norm;
  * "swapped":           s_a and s_m exchanged;
  * "depth_by_L":        an initialisation mutant (init_params): CaiT's rule, one value for every layer chosen by the
                         total depth L instead of each layer's own depth.
and of stable (stable_mutate):
  * "max_abs":           m = max_c |x[c]|;
  * "norm_then_divide":  hf = LN_f(x) / m, the division after the norm;
  * "grad_through_max":  m not detached: the gradient flows through the maximum;
  * "no_shrink":         the embedding gradients not shrunk.
"""
import math

import torch

from . import dalle_gelu as OG
from . import dalle_glu as OGL
from . import dalle_gmlp as OM
from . import dalle_shift as OS
from .dalle import Quirks, _r, layer_norm, shift_labels
from .dalle_rotary import rotate

MUTATIONS = ("post_residual", "scale_before_norm", "swapped", "depth_by_L")
STABLE_MUTATIONS = ("max_abs", "norm_then_divide", "grad_through_max", "no_shrink")
ALPHA = 0.1


class _GradScale(torch.autograd.Function):
    """Identity forward, gradient times alpha: tokens * alpha + tokens.detach() * (1 - alpha) without its rounding."""

    @staticmethod
    def forward(ctx, x, alpha):
        ctx.alpha = alpha
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g * ctx.alpha, None


def divide_max(x, mutate=None):
    """DivideMax of the rows of x: (x / m, m) with m the detached row maximum (mutants as the module doc)."""
    m = x.abs().amax(-1, keepdim=True) if mutate == "max_abs" else x.amax(-1, keepdim=True)
    if mutate != "grad_through_max":
        m = m.detach()
    return x / m, m


def depth_value(n):
    """DALLE-pytorch's initial LayerScale value at 1-based depth n."""
    return 0.1 if n <= 18 else 1e-5 if n <= 24 else 1e-6


def scale_names(cfg):
    """The LayerScale variables of every layer in layout order: the token mixer's, then the MLP's."""
    out = []
    for l in range(cfg.n_layers):
        pre = f"layer_{l}/"
        out += [pre + ("gmlp" if OM.is_mlp(cfg, l) else "attn") + "/layer_scale", pre + "mlp/layer_scale"]
    return out


def init_params(params, cfg, value=True, seed=None, mutate=None):
    """params with the LayerScale vectors added.  seed None: the initial values of `value` (True: by depth, a number:
    that number); mutate "depth_by_L": every layer gets depth_value(L).  With a seed each entry is drawn from
    U(0.3, 0.9), so that every channel and both branches differ."""
    out = dict(params)
    g = torch.Generator().manual_seed(0 if seed is None else seed)
    d, Lyr = cfg.n_embd, cfg.n_layers
    names = scale_names(cfg)
    for l in range(Lyr):
        if seed is not None:
            v = None
        elif mutate == "depth_by_L":
            v = depth_value(Lyr)
        else:
            v = depth_value(l + 1) if value is True else float(value)
        for name in names[2 * l:2 * l + 2]:
            out[name] = torch.full((d,), v) if v is not None else 0.3 + 0.6 * torch.rand(d, generator=g)
    return out


def check(mutate, sandwich_norm, layer_scale):
    if mutate is None:
        return
    if mutate not in MUTATIONS or mutate == "depth_by_L":
        raise ValueError(f"mutation {mutate!r} is not one of the forward mutations {MUTATIONS[:3]}")
    if not layer_scale or (mutate == "scale_before_norm" and not sandwich_norm):
        raise ValueError(f"mutation {mutate!r} needs layer_scale (and scale_before_norm the sandwich LayerNorm)")


def forward(params, tokens, cfg, dropout=None, bf16=False, quirks: Quirks = None, activation="relu", gated=False,
            layers=None, rotary=None, shift_tokens=False, sandwich_norm=False, layer_scale=False, stable=False,
            gmlp_mutate=None, scale_mutate=None, stable_mutate=None):
    """oracle/dalle_gmlp.forward with LayerScale on both branches of every layer (layer_scale=False: without it) and
    DALLE-pytorch's stable option (stable=False: without it): returns (loss, loss_batch, logits).  dropout: None or
    (rates, seed, step, row0)."""
    OM.check(gmlp_mutate)
    check(scale_mutate, sandwich_norm, layer_scale)
    if stable_mutate is not None and (stable_mutate not in STABLE_MUTATIONS or not stable):
        raise ValueError(f"stable mutation {stable_mutate!r} is not one of {STABLE_MUTATIONS}, or stable is off")
    OGL.check(activation, None)
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
    sh = (lambda t: t) if not shift_tokens else (lambda t: OS.shift(t, TL, Wg, None))
    names = scale_names(cfg)

    def norm(x, name):
        return sh(_r(layer_norm(x, W(name + "/g"), W(name + "/b"), q_.ln_eps), bf16))

    def residual(x, o, mask, name, scale):
        """x + drop(o), or with the sandwich LayerNorm x + LN_name(drop(o)), one rounding (as oracle/dalle_gmlp);
        with LayerScale what is added is multiplied by the vector `scale` first."""
        if mask is not None:
            o = _r(o * mask, bf16)
        s = W(scale) if layer_scale else None
        if sandwich_norm:
            if scale_mutate == "scale_before_norm":
                o = o * s
                s = None
            v = layer_norm(o, W(name + "/g"), W(name + "/b"), q_.ln_eps)
        else:
            v = o
        if s is None:
            return _r(x + v, bf16)
        if scale_mutate == "post_residual":
            return _r((x + v) * s, bf16)
        return _r(x + s * v, bf16)

    x = _r(drop(W("embedding/wte")[tokens], dm["wte"]) + drop(W("positional_embedding/wpe")[:S], dm["wpe"]), bf16)
    if stable and stable_mutate != "no_shrink":
        x = _GradScale.apply(x, ALPHA)
    for l in range(cfg.n_layers):
        pfx = f"layer_{l}/"
        s_a, s_m = names[2 * l:2 * l + 2]
        if scale_mutate == "swapped":
            s_a, s_m = s_m, s_a
        h = norm(x, pfx + "norm_1")
        if OM.is_mlp(cfg, l):
            a = OM.gmlp_branch(h, params, pfx, q_.ln_eps, bf16, gmlp_mutate)
        else:
            mask = layers.attention_mask(cfg, l, S, q_)
            q = rot(_r(h @ W(pfx + "attn/q"), bf16).view(B, S, H, dh))
            k = rot(_r(h @ W(pfx + "attn/k"), bf16).view(B, S, H, dh))
            v = _r(h @ W(pfx + "attn/v"), bf16).view(B, S, H, dh)
            logits = torch.einsum("bihe,bjhe->bhij", q, k) * q_.attn_scale + mask              # fp32 ‡
            p = _r(drop(torch.softmax(logits, dim=-1), dm["attn"][l]), bf16)
            a = _r(torch.einsum("bhij,bjhe->bihe", p, v).reshape(B, S, H * dh), bf16)
            a = _r(a @ W(pfx + "attn/o") + W(pfx + "attn/compute_output_bias/o_b"), bf16)
        x = residual(x, a, dm["attn_out"][l], pfx + "attn/norm_out", s_a)
        h = norm(x, pfx + "norm_2")
        y = h @ W(pfx + "mlp/mlp_linear_1/kernel") + W(pfx + "mlp/mlp_linear_1/bias")
        if gated:
            h1 = OGL.gated_mlp(y, activation, bf16, None)
        else:
            h1 = _r(OG.mlp_activation(y, activation, bf16), bf16)
        h2 = _r(h1 @ W(pfx + "mlp/mlp_linear_2/kernel") + W(pfx + "mlp/mlp_linear_2/bias"), bf16)
        x = residual(x, h2, dm["mlp_out"][l], pfx + "mlp/norm_out", s_m)
    if stable and stable_mutate == "norm_then_divide":
        hf = _r(layer_norm(x, W("to_logits/layer_norm/g"), W("to_logits/layer_norm/b"), q_.ln_eps) /
                divide_max(x)[1], bf16)
    else:
        u = divide_max(x, stable_mutate)[0] if stable else x
        hf = _r(layer_norm(u, W("to_logits/layer_norm/g"), W("to_logits/layer_norm/b"), q_.ln_eps), bf16)
    logits = hf @ W("to_logits/linear_out/kernel") + W("to_logits/linear_out/bias")
    logits = logits.to(torch.promote_types(logits.dtype, torch.float32))
    labels = shift_labels(tokens, cfg.eos_token_id)
    loss_batch = torch.logsumexp(logits, -1) - logits.gather(-1, labels[..., None]).squeeze(-1)
    return loss_batch.mean(), loss_batch, logits


def loss_and_grads(params, tokens, cfg, **kw):
    """Autograd of forward(): (loss, loss_batch, logits, grads)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, loss_batch, logits = forward(leaves, tokens, cfg, **kw)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads
