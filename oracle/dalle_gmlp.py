"""ORACLE (test infrastructure, NOT product code) — the DALL-E transformer with gMLP token-mixing layers.

DALLE-pytorch's attention type 'mlp' is the gMLP block of "Pay Attention to MLPs" (its gMLPBlock(dim=d, dim_ff=4d,
seq_len=S, causal=True), one head).  In a layer whose type is "mlp", the pre-norm branch computes, in place of
attention, with C = 2d:

    z          = bf16(LN1(x) W_in + b_in)                 layer_l/gmlp/proj_in/{kernel,bias}, W_in [d, 4d]
    u          = bf16(gelu(z))                            mtf's tanh GELU (DALLE-pytorch uses the erf nn.GELU)
    res, gate  = u[:, :C], u[:, C:]
    gn         = bf16(LN_sgu(gate))                       layer_l/gmlp/sgu/norm/{g,b}, eps = ln_eps
    mixed[b,i] = sum_{j <= i} W_sgu[i, j] gn[b, j] + c_sgu[i]     fp32; layer_l/gmlp/sgu/{weight,bias}, W_sgu [S, S]
    h          = bf16(mixed res)
    o          = bf16(h W_out + b_out)                    layer_l/gmlp/proj_out/{kernel,bias}, W_out [C, d]

and o takes the attention output's place: residual dropout, the sandwich LayerNorm LNa (layer_l/attn/norm_out) and
the residual add are unchanged, as is the layer's MLP branch.  Rotary embeddings and attention dropout do not touch the
layer.  W_sgu's strict upper triangle is zero (the engine keeps it so); this oracle masks it with tril all the same,
so that the "unmasked" mutant differs where a test puts non-zeros there.

forward() is oracle/dalle_sandwich.forward with the gMLP layers added; a model without them computes bit for bit what
that forward computes (tests/test_mlp_layers_cpu.py).  Mutations a correct engine must fail:
  * "unmasked": W_sgu used without the causal mask;
  * "no_norm":  gn = gate (the SGU LayerNorm skipped);
  * "col_bias": c_sgu added along the channels (c_sgu[k mod S] to channel k) instead of per position;
  * "swapped":  res and gate exchanged (the first half gated, the second normalised and mixed);
  * "erf_gelu": u from PyTorch's erf GELU instead of the tanh form.
"""
import math

import torch

from . import dalle_gelu as OG
from . import dalle_glu as OGL
from . import dalle_shift as OS
from .dalle import Quirks, _r, layer_norm, shift_labels
from .dalle_rotary import rotate

MUTATIONS = ("unmasked", "no_norm", "col_bias", "swapped", "erf_gelu")
GMLP_VARS = ("proj_in/kernel", "proj_in/bias", "sgu/norm/g", "sgu/norm/b", "sgu/weight", "sgu/bias",
             "proj_out/kernel", "proj_out/bias")


def is_mlp(cfg, layer):
    types = getattr(cfg, "attention_types", None)
    return types is not None and types[layer] == "mlp"


def init_params(params, cfg, seed=None):
    """params with every "mlp" layer's attention variables replaced by the gMLP block's.  seed None: the engine's
    initialisation (W_in ~ N(0, 0.02), W_out ~ N(0, 0.02 / sqrt(L)), W_sgu ~ U(-1e-3/S, 1e-3/S) lower triangular,
    c_sgu = 1, norm g = 1, biases 0).  With a seed every variable is drawn so that each piece of the block moves the
    output: W_in ~ N(0, 1 / d), W_out ~ N(0, 1 / 2d), W_sgu ~ N(0, 1 / (i + 1)) in row i (lower triangle), c_sgu ~
    1 + 0.3 N, g ~ 1 + 0.3 N, biases ~ 0.1 N."""
    out = dict(params)
    d, S, Lyr = cfg.n_embd, cfg.seq_len, cfg.n_layers
    C = 2 * d
    g = torch.Generator().manual_seed(0 if seed is None else seed)
    for l in range(Lyr):
        if not is_mlp(cfg, l):
            continue
        pre = f"layer_{l}/"
        for v in ("q", "k", "v", "o", "compute_output_bias/o_b"):
            out.pop(pre + "attn/" + v, None)
        gp = pre + "gmlp/"
        out[gp + "proj_in/kernel"] = torch.randn(d, 4 * d, generator=g) * 0.02
        out[gp + "proj_out/kernel"] = torch.randn(C, d, generator=g) * (0.02 / math.sqrt(Lyr))
        if seed is None:
            eps = 1e-3 / S
            out[gp + "sgu/weight"] = torch.tril((torch.rand(S, S, generator=g) * 2 - 1) * eps)
            out[gp + "sgu/bias"] = torch.ones(S)
            out[gp + "sgu/norm/g"], out[gp + "sgu/norm/b"] = torch.ones(C), torch.zeros(C)
            out[gp + "proj_in/bias"], out[gp + "proj_out/bias"] = torch.zeros(4 * d), torch.zeros(d)
        else:
            rows = torch.arange(S, dtype=torch.float32)[:, None] + 1
            out[gp + "sgu/weight"] = torch.tril(torch.randn(S, S, generator=g) / rows.sqrt())
            out[gp + "sgu/bias"] = 1 + 0.3 * torch.randn(S, generator=g)
            out[gp + "sgu/norm/g"] = 1 + 0.3 * torch.randn(C, generator=g)
            out[gp + "sgu/norm/b"] = 0.1 * torch.randn(C, generator=g)
            out[gp + "proj_in/bias"] = 0.1 * torch.randn(4 * d, generator=g)
            out[gp + "proj_out/bias"] = 0.1 * torch.randn(d, generator=g)
            out[gp + "proj_out/kernel"] = torch.randn(C, d, generator=g) * C ** -0.5
            out[gp + "proj_in/kernel"] = torch.randn(d, 4 * d, generator=g) * d ** -0.5
    return out


def check(mutate):
    if mutate is not None and mutate not in MUTATIONS:
        raise ValueError(f"mutation {mutate!r} is not one of {MUTATIONS}")


def sgu(u, g, b, w, c, eps, bf16=False, mutate=None):
    """The spatial gating unit on u [B, n, 2C] (GELU output, bf16 values): (h, mixed) with mixed in fp32."""
    B, n, C2 = u.shape
    C = C2 // 2
    res, gate = (u[..., C:], u[..., :C]) if mutate == "swapped" else (u[..., :C], u[..., C:])
    gn = gate if mutate == "no_norm" else _r(layer_norm(gate, g, b, eps), bf16)
    w = w[:n, :n]
    if mutate != "unmasked":
        w = torch.tril(w)
    mixed = torch.einsum("ij,bjc->bic", w, gn)
    if mutate == "col_bias":
        mixed = mixed + c[torch.arange(C) % c.numel()]
    else:
        mixed = mixed + c[:n, None]
    return _r(mixed * res, bf16), mixed


def gmlp_branch(h, params, pfx, eps, bf16=False, mutate=None):
    """The gMLP block on the LN1 output h [B, n, d]: o = bf16(h' W_out + b_out) before residual dropout."""
    W = (lambda n: _r(params[n], bf16))
    gp = pfx + "gmlp/"
    z = _r(h @ W(gp + "proj_in/kernel") + W(gp + "proj_in/bias"), bf16)
    u = _r(torch.nn.functional.gelu(z) if mutate == "erf_gelu" else OG.gelu(z), bf16)
    hh, _ = sgu(u, W(gp + "sgu/norm/g"), W(gp + "sgu/norm/b"), W(gp + "sgu/weight"), W(gp + "sgu/bias"), eps, bf16,
                mutate)
    return _r(hh @ W(gp + "proj_out/kernel") + W(gp + "proj_out/bias"), bf16)


def forward(params, tokens, cfg, dropout=None, bf16=False, quirks: Quirks = None, activation="relu", gated=False,
            layers=None, rotary=None, shift_tokens=False, sandwich_norm=False, gmlp_mutate=None):
    """DALLE.forward (src/dalle_mtf/models.py:397-416) with gMLP layers where cfg.attention_types says "mlp", on top of
    oracle/dalle_sandwich.forward's options (sandwich_norm=False: without the sandwich LayerNorm): returns (loss,
    loss_batch, logits).  dropout: None or (rates, seed, step, row0)."""
    check(gmlp_mutate)
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

    def norm(x, name):
        return sh(_r(layer_norm(x, W(name + "/g"), W(name + "/b"), q_.ln_eps), bf16))

    def residual(x, o, mask, name):
        """x + drop(o), or with the sandwich LayerNorm x + LN_name(drop(o)), one rounding (as oracle/dalle_sandwich)."""
        if mask is not None:
            o = _r(o * mask, bf16)
        if not sandwich_norm:
            return _r(x + o, bf16)
        return _r(x + layer_norm(o, W(name + "/g"), W(name + "/b"), q_.ln_eps), bf16)

    x = _r(drop(W("embedding/wte")[tokens], dm["wte"]) + drop(W("positional_embedding/wpe")[:S], dm["wpe"]), bf16)
    for l in range(cfg.n_layers):
        pfx = f"layer_{l}/"
        h = norm(x, pfx + "norm_1")
        if is_mlp(cfg, l):
            a = gmlp_branch(h, params, pfx, q_.ln_eps, bf16, gmlp_mutate)
        else:
            mask = layers.attention_mask(cfg, l, S, q_)
            q = rot(_r(h @ W(pfx + "attn/q"), bf16).view(B, S, H, dh))
            k = rot(_r(h @ W(pfx + "attn/k"), bf16).view(B, S, H, dh))
            v = _r(h @ W(pfx + "attn/v"), bf16).view(B, S, H, dh)
            logits = torch.einsum("bihe,bjhe->bhij", q, k) * q_.attn_scale + mask              # fp32 ‡
            p = _r(drop(torch.softmax(logits, dim=-1), dm["attn"][l]), bf16)
            a = _r(torch.einsum("bhij,bjhe->bihe", p, v).reshape(B, S, H * dh), bf16)
            a = _r(a @ W(pfx + "attn/o") + W(pfx + "attn/compute_output_bias/o_b"), bf16)
        x = residual(x, a, dm["attn_out"][l], pfx + "attn/norm_out")
        h = norm(x, pfx + "norm_2")
        y = h @ W(pfx + "mlp/mlp_linear_1/kernel") + W(pfx + "mlp/mlp_linear_1/bias")
        if gated:
            h1 = OGL.gated_mlp(y, activation, bf16, None)
        else:
            h1 = _r(OG.mlp_activation(y, activation, bf16), bf16)
        h2 = _r(h1 @ W(pfx + "mlp/mlp_linear_2/kernel") + W(pfx + "mlp/mlp_linear_2/bias"), bf16)
        x = residual(x, h2, dm["mlp_out"][l], pfx + "mlp/norm_out")
    hf = _r(layer_norm(x, W("to_logits/layer_norm/g"), W("to_logits/layer_norm/b"), q_.ln_eps), bf16)
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
