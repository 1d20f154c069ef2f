"""ORACLE (test infrastructure, NOT product code) — the DALL-E transformer with the MLP nonlinearity as a parameter.

The reference's DALLE takes an activation_fn (src/dalle_mtf/models.py:146,177-179, applied in mlp() at :320) whose
default is mtf.relu.  GPT-Neo's configs select GELU with "activation_function": "gelu"; mtf's GELU is the tanh form
(‡ recalled mtf 0.1.18 behaviour, as in oracle/dalle.py):

    gelu(x) = 0.5 x (1 + tanh(u)) = x sigma(2u),   u = sqrt(2/pi) (x + 0.044715 x^3)

which equals torch.nn.functional.gelu(x, approximate="tanh").

Cast points (bf16): mtf's dense layer returns the activation dtype, so the pre-activation z = bf16(x W1 + b1) is
rounded before the nonlinearity and h = bf16(act(z)); autograd then also rounds dZ = bf16(dH act'(z)) at z's cast.
For ReLU both roundings give the same values (max(bf16(y), 0) = bf16(max(y, 0)) up to the sign of a zero, and a bf16
dH times a 0/1 mask is already bf16).

forward() is the forward of oracle/dalle_local.py (which with every layer global is operation for operation the
forward of oracle/dalle.py and, with dropout, of oracle/dalle_dropout.py) with the MLP written as
_r(mlp_activation(x W1 + b1, activation, bf16, mutate), bf16).  The activation, the mutation and bf16 are explicit
arguments; the attention layers come from `layers`, a module with attention_mask(cfg, layer, S, quirks) and
dropout_masks(dropout, B, cfg) (oracle.dalle_local by default, the axial / conv oracles of tests/ for their configs).
With activation "relu" it computes bit for bit what each of those forwards computes (tests/test_gelu_cpu.py).
"""
import dataclasses
import math

import torch

from . import dalle_local
from .dalle import DalleConfig, Quirks, _r, layer_norm, shift_labels

ACTIVATIONS = ("relu", "gelu")
GELU_CUBIC = 0.044715
SQRT_2_OVER_PI = math.sqrt(2.0 / math.pi)
# mutation: GELU without its cubic term (at x = 2 gelu changes by about 0.03); a correct kernel must fail against it
MUTATIONS = ("gelu_no_cubic",)


def gelu(z, cubic=GELU_CUBIC):
    """mtf's tanh GELU in z's dtype (differentiable), as z sigma(2u): 1 + tanh(u) would cancel in the negative tail."""
    return z * torch.sigmoid(2.0 * SQRT_2_OVER_PI * (z + cubic * z * z * z))


def gelu_grad(z, cubic=GELU_CUBIC):
    """Closed-form d gelu / dz = s + z s (1 - s) 2 sqrt(2/pi) (1 + 3 cubic z^2), s = sigma(2u)."""
    s = torch.sigmoid(2.0 * SQRT_2_OVER_PI * (z + cubic * z * z * z))
    return s + z * s * (1.0 - s) * 2.0 * SQRT_2_OVER_PI * (1.0 + 3.0 * cubic * z * z)


def check(activation, mutate=None):
    if activation not in ACTIVATIONS:
        raise ValueError(f"activation must be one of {ACTIVATIONS}, got {activation!r}")
    if mutate is not None and (activation != "gelu" or mutate not in MUTATIONS):
        raise ValueError(f"mutation {mutate!r} is not one of {MUTATIONS} of GELU")


def mlp_activation(y, name="relu", bf16=False, mutate=None):
    """The MLP nonlinearity applied to the pre-activation y = x W1 + b1 with the cast points above (the caller rounds
    the result to bf16)."""
    check(name, mutate)
    z = _r(y, bf16)
    if name == "relu":
        return torch.relu(z)
    return gelu(z, 0.0 if mutate == "gelu_no_cubic" else GELU_CUBIC)


def _layers(cfg, layers):
    """(config with per-layer types, module of its attention masks)."""
    if layers is not None:
        return cfg, layers
    if type(cfg) is DalleConfig:          # every layer global: the local oracle's config without local layers
        return dalle_local.LocalConfig(**dataclasses.asdict(cfg)), dalle_local
    if type(cfg) is dalle_local.LocalConfig:
        return cfg, dalle_local
    raise ValueError(f"{type(cfg).__name__}: pass the module of its attention masks as layers=")


def forward(params, tokens, cfg: DalleConfig, dropout=None, bf16=False, quirks: Quirks = None, activation="relu",
            mutate=None, layers=None):
    """DALLE.forward (src/dalle_mtf/models.py:397-416) with MLP nonlinearity `activation`: returns (loss, loss_batch,
    logits).  dropout: None (mode "eval") or (rates, seed, step, row0) as oracle.dalle_dropout.forward takes it."""
    check(activation, mutate)
    cfg, layers = _layers(cfg, layers)
    q_ = quirks or Quirks()
    B, S = tokens.shape
    H, dh = cfg.n_heads, cfg.head_dim
    W = (lambda n: _r(params[n], bf16))
    none = [None] * cfg.n_layers
    dm = layers.dropout_masks(dropout, B, cfg) if dropout is not None else \
        {"wte": None, "wpe": None, "attn": none, "attn_out": none, "mlp_out": none}
    drop = (lambda t, m: t if m is None else t * m)
    x = _r(drop(W("embedding/wte")[tokens], dm["wte"]) + drop(W("positional_embedding/wpe")[:S], dm["wpe"]), bf16)
    for l in range(cfg.n_layers):
        pre = f"layer_{l}/"
        mask = layers.attention_mask(cfg, l, S, q_)
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
        y = h @ W(pre + "mlp/mlp_linear_1/kernel") + W(pre + "mlp/mlp_linear_1/bias")
        h1 = _r(mlp_activation(y, activation, bf16, mutate), bf16)                         # :320
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


def loss_and_grads(params, tokens, cfg, dropout=None, bf16=False, quirks=None, activation="relu", mutate=None,
                   layers=None):
    """Autograd of forward() (mtf.gradients, src/optimizers.py:34): (loss, loss_batch, logits, grads)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, loss_batch, logits = forward(leaves, tokens, cfg, dropout, bf16=bf16, quirks=quirks, activation=activation,
                                       mutate=mutate, layers=layers)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads
