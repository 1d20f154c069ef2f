"""ORACLE (test infrastructure, NOT product code) — DALLE-pytorch's parameter sharing around the existing forwards.

DALLE-pytorch's DALLE(...) takes three sharing options (recalled, not checked):
  * share_input_output_emb: SharedEmbedding takes the input embedding's rows from the output projection's weight, so
    logits = hf wte^T + bout with one [V, d] table; the bias stays.  With `stable`, the 0.1 gradient shrink sits on
    the embedding output (tokens * 0.1 + tokens.detach() * 0.9), so it scales the gathered rows' gradient only, never
    the logits path's.
  * shared_attn_ids / shared_ff_ids: lists of ids cycled to the depth (cycle([0, 1]) at 6 layers: 0 1 0 1 0 1); layers
    with the same id use one attention (or gMLP) module / one feed-forward module.  Each layer wraps it in its own
    PreNorm and LayerScale, so LayerNorms (the sandwich ones too) and scales are never shared.  Layers sharing an
    attention id must have the same attention type.

Here a shared model's variables are those of an unshared twin minus, per layer, the module variables of every layer
that is not its module's owner (the lowest layer with its id), and minus to_logits/linear_out/kernel when tied
(names()).  expand() rebuilds the full per-layer dict the existing oracle forwards take, every user of a module
holding the *same* leaf tensor and to_logits/linear_out/kernel = wte[:V]^T, so that autograd sums every use's
gradient.  With every id distinct and no tying it returns its input, and the forwards compute bit for bit what they
compute without it.

Mutations a correct engine must fail (MUTATIONS):
  * "untied_grad":   the output projection's part of the wte gradient dropped (wte detached on the logits path);
  * "shrink_output": stable's 0.1 shrink also applied to that part;
  * "shared_norms":  the users' LayerNorms (norm_1 with the token mixer, norm_2 with the MLP) shared with the module;
  * "last_owner":    the module initialised and named at its last user instead of its first;
  * "no_cycle":      the ids not cycled: a layer past the end of the list keeps its own module.
"""
import torch

from . import dalle_gmlp as OM
from . import dalle_layer_scale as OLS

MUTATIONS = ("untied_grad", "shrink_output", "shared_norms", "last_owner", "no_cycle")
OUT_KERNEL = "to_logits/linear_out/kernel"
ATTN_VARS = ("attn/q", "attn/k", "attn/v", "attn/o", "attn/compute_output_bias/o_b")
GMLP_VARS = tuple("gmlp/" + v for v in OM.GMLP_VARS)
FF_VARS = ("mlp/mlp_linear_1/kernel", "mlp/mlp_linear_1/bias", "mlp/mlp_linear_2/kernel", "mlp/mlp_linear_2/bias")


def check(mutate):
    if mutate is not None and mutate not in MUTATIONS:
        raise ValueError(f"mutation {mutate!r} is not one of {MUTATIONS}")


def layer_ids(ids, n_layers, mutate=None):
    """The per-layer ids: `ids` cycled to n_layers (None: every layer its own; "no_cycle": past the list, too)."""
    if ids is None:
        return [("own", i) for i in range(n_layers)]
    if mutate == "no_cycle":
        return [ids[i] if i < len(ids) else ("own", i) for i in range(n_layers)]
    return [ids[i % len(ids)] for i in range(n_layers)]


def owners(ids, n_layers, mutate=None):
    """Per layer, the layer whose module it uses: the lowest with the same id ("last_owner": the highest)."""
    per = layer_ids(ids, n_layers, mutate)
    users = {}
    for i, v in enumerate(per):
        users.setdefault(v, []).append(i)
    pick = max if mutate == "last_owner" else min
    return [pick(users[v]) for v in per]


def mixer_vars(cfg, layer):
    """The token mixer's variables (below layer_{layer}/) of layer `layer`: a gMLP block's or attention's."""
    return GMLP_VARS if OM.is_mlp(cfg, layer) else ATTN_VARS


def names(full_names, cfg, tie=False, attn_ids=None, ff_ids=None, mutate=None):
    """The variables of the shared model, in the order of full_names (an unshared twin's variables)."""
    ao, fo = owners(attn_ids, cfg.n_layers, mutate), owners(ff_ids, cfg.n_layers, mutate)
    drop = {OUT_KERNEL} if tie else set()
    for l in range(cfg.n_layers):
        if ao[l] != l:
            drop |= {f"layer_{l}/{v}" for v in mixer_vars(cfg, l)}
        if fo[l] != l:
            drop |= {f"layer_{l}/{v}" for v in FF_VARS}
    return [n for n in full_names if n not in drop]


def share(params, cfg, tie=False, attn_ids=None, ff_ids=None, mutate=None):
    """The shared model's variables taken from an unshared twin's dict: each module from its owner's entries."""
    return {k: params[k] for k in names(list(params), cfg, tie, attn_ids, ff_ids, mutate)}


def expand(params, cfg, tie=False, attn_ids=None, ff_ids=None, mutate=None):
    """The full per-layer dict of a shared model's variables: every user of a module gets its owner's tensors (the same
    objects), and a tied model's to_logits/linear_out/kernel is wte^T."""
    check(mutate)
    full = dict(params)
    ao, fo = owners(attn_ids, cfg.n_layers, mutate), owners(ff_ids, cfg.n_layers, mutate)
    for l in range(cfg.n_layers):
        for own, vars_, norm in ((ao[l], mixer_vars(cfg, l), "norm_1"), (fo[l], FF_VARS, "norm_2")):
            if own == l:
                continue
            extra = (norm + "/g", norm + "/b") if mutate == "shared_norms" else ()
            for v in vars_ + extra:
                full[f"layer_{l}/{v}"] = params[f"layer_{own}/{v}"]
    if tie:
        wte = params["embedding/wte"]
        if mutate == "untied_grad":
            wte = wte.detach()
        elif mutate == "shrink_output":
            wte = OLS._GradScale.apply(wte, OLS.ALPHA)
        full[OUT_KERNEL] = wte.t()
    return full


def wrap(forward, cfg, tie=False, attn_ids=None, ff_ids=None, mutate=None):
    """forward(params, ...) of a shared model: `forward` (an oracle forward over full dicts) after expand()."""
    return lambda params, *a, **k: forward(expand(params, cfg, tie, attn_ids, ff_ids, mutate), *a, **k)


def loss_and_grads(params, tokens, cfg, tie=False, attn_ids=None, ff_ids=None, mutate=None, forward=OLS.forward,
                   **kw):
    """Autograd of a shared model whose variables are taken from `params` (an unshared twin's, or already shared:
    share() keeps what it needs): (loss, loss_batch, logits, grads), grads keyed by the shared model's names."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in share(params, cfg, tie, attn_ids, ff_ids, mutate).items()}
    loss, loss_batch, logits = wrap(forward, cfg, tie, attn_ids, ff_ids, mutate)(leaves, tokens, cfg, **kw)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads
