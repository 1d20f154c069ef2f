"""ORACLE (test infrastructure, NOT product code) — the DALL-E transformer with a gated MLP (GLU).

DALLE-pytorch's FeedForward is always gated: Linear(dim, 2 * mult * dim), then `x, gates = x.chunk(2, dim=-1)` and
`x * act(gates)`, then Linear(mult * dim, dim) with mult = 4 (T5.1.1's "gated-gelu" is the same block).  With the
config key "gated_mlp": true the engine builds that MLP, with the value half first and the gate half second as
chunk(2) splits them:

    y      = LN2(x) W1 + b1                     W1 [d, 8d], b1 [8d]
    zv, zg = bf16(y[:, :4d]), bf16(y[:, 4d:])
    a      = bf16(act(zg))                      act = the activation_function: relu (ReGLU) or mtf's tanh gelu (GEGLU)
    h      = bf16(zv a)
    out    = h W2 + b2                          W2 [4d, d]

Cast points as in oracle/dalle_gelu.py (`_r` at each bf16 cast); autograd rounds each gradient at its cast.

forward() is oracle/dalle_gelu.forward (the attention layers from `layers`, the local oracle by default) with that
MLP, and with q and k rotated as oracle/dalle_rotary.forward rotates them when `rotary` = (r, base) is given.
gated=False gives oracle/dalle_gelu.forward's MLP, bit for bit (tests/test_gated_mlp_cpu.py).  Mutations a correct
engine must fail:
  * "swap":    the nonlinearity on the first half instead of the second;
  * "shift64": value column j paired with gate column (j + 64) mod 4d (a tile-pairing bug of the fused epilogue).
"""
import torch

from . import dalle_gelu as OG
from .dalle import Quirks, _r, layer_norm, shift_labels
from .dalle_rotary import rotate

MUTATIONS = ("swap", "shift64")


def check(activation, mutate=None):
    OG.check(activation)
    if mutate is not None and mutate not in MUTATIONS:
        raise ValueError(f"mutation {mutate!r} is not one of {MUTATIONS}")


def act(z, name):
    return torch.relu(z) if name == "relu" else OG.gelu(z)


def gated_mlp(y, name="relu", bf16=False, mutate=None):
    """h = bf16(zv bf16(act(zg))) of the pre-activation y = x W1 + b1 ([..., 8d], value half first)."""
    check(name, mutate)
    n = y.shape[-1] // 2
    zv, zg = _r(y[..., :n], bf16), _r(y[..., n:], bf16)
    if mutate == "swap":
        zv, zg = zg, zv
    elif mutate == "shift64":
        zg = torch.roll(zg, -64, dims=-1)          # column j reads gate column (j + 64) mod n
    return _r(zv * _r(act(zg, name), bf16), bf16)


def forward(params, tokens, cfg, dropout=None, bf16=False, quirks: Quirks = None, activation="relu", gated=True,
            mutate=None, layers=None, rotary=None):
    """DALLE.forward (src/dalle_mtf/models.py:397-416) with the gated MLP above (gated=False: the ungated MLP of
    oracle/dalle_gelu.py): returns (loss, loss_batch, logits).  dropout: None or (rates, seed, step, row0)."""
    check(activation, mutate)
    if mutate is not None and not gated:
        raise ValueError("the mutations are of the gated MLP")
    cfg, layers = OG._layers(cfg, layers)
    q_ = quirks or Quirks()
    B, S = tokens.shape
    H, dh = cfg.n_heads, cfg.head_dim
    W = (lambda n: _r(params[n], bf16))
    none = [None] * cfg.n_layers
    dm = layers.dropout_masks(dropout, B, cfg) if dropout is not None else \
        {"wte": None, "wpe": None, "attn": none, "attn_out": none, "mlp_out": none}
    drop = (lambda t, m: t if m is None else t * m)
    rot = (lambda t: t) if rotary is None else (lambda t: _r(rotate(t, rotary[0], rotary[1]), bf16))
    x = _r(drop(W("embedding/wte")[tokens], dm["wte"]) + drop(W("positional_embedding/wpe")[:S], dm["wpe"]), bf16)
    for l in range(cfg.n_layers):
        pre = f"layer_{l}/"
        mask = layers.attention_mask(cfg, l, S, q_)
        h = _r(layer_norm(x, W(pre + "norm_1/g"), W(pre + "norm_1/b"), q_.ln_eps), bf16)
        q = rot(_r(h @ W(pre + "attn/q"), bf16).view(B, S, H, dh))
        k = rot(_r(h @ W(pre + "attn/k"), bf16).view(B, S, H, dh))
        v = _r(h @ W(pre + "attn/v"), bf16).view(B, S, H, dh)
        logits = torch.einsum("bihe,bjhe->bhij", q, k) * q_.attn_scale + mask              # fp32 ‡
        p = _r(drop(torch.softmax(logits, dim=-1), dm["attn"][l]), bf16)
        a = _r(torch.einsum("bhij,bjhe->bihe", p, v).reshape(B, S, H * dh), bf16)
        a = _r(a @ W(pre + "attn/o") + W(pre + "attn/compute_output_bias/o_b"), bf16)
        if dm["attn_out"][l] is not None:
            a = _r(a * dm["attn_out"][l], bf16)
        x = _r(x + a, bf16)
        h = _r(layer_norm(x, W(pre + "norm_2/g"), W(pre + "norm_2/b"), q_.ln_eps), bf16)
        y = h @ W(pre + "mlp/mlp_linear_1/kernel") + W(pre + "mlp/mlp_linear_1/bias")
        if gated:
            h1 = gated_mlp(y, activation, bf16, mutate)
        else:
            h1 = _r(OG.mlp_activation(y, activation, bf16), bf16)
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


def init_params(params, cfg, seed):
    """A copy of an ungated parameter dict whose W1 / b1 are widened to [d, 8d] / [8d] by a second normal(0.02)
    gate half (drawn from `seed`), so that an oracle config's params serve the gated model."""
    g = torch.Generator().manual_seed(seed)
    out = dict(params)
    for l in range(cfg.n_layers):
        k, b = f"layer_{l}/mlp/mlp_linear_1/kernel", f"layer_{l}/mlp/mlp_linear_1/bias"
        out[k] = torch.cat([params[k], torch.randn(params[k].shape, generator=g) * 0.02], 1)
        out[b] = torch.cat([params[b], torch.zeros(params[b].shape)])
    return out


def loss_and_grads(params, tokens, cfg, dropout=None, bf16=False, quirks=None, activation="relu", gated=True,
                   mutate=None, layers=None, rotary=None):
    """Autograd of forward(): (loss, loss_batch, logits, grads)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, loss_batch, logits = forward(leaves, tokens, cfg, dropout, bf16=bf16, quirks=quirks, activation=activation,
                                       gated=gated, mutate=mutate, layers=layers, rotary=rotary)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads
