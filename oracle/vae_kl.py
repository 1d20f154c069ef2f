"""ORACLE (test infrastructure, NOT product code) — the discrete VAE's optional KL term (an extension: the reference has
no KL term; DESIGN.md §4), on top of oracle/vae.py, which it leaves as it is.

  KL_r = sum_k q_rk (l_rk - lse_r) + log K = KL(q_r || Uniform(K)),  q_r = softmax(l_r), l_r the raw encoder logits of
  latent row r (no Gumbel noise, no temperature);  KL = mean over the latent rows;  loss = MSE + beta_t * KL.

Mutation switches (`mutate`), for tests that must tell the engine apart from plausible mistakes:
  "noisy_logits"   KL of the softmax of the Gumbel-noised, tempered logits (logits + g) / tau instead of the raw ones;
  "no_centring"    the KL gradient without its centring term: c q (l - lse) instead of c q (l - lse - e);
  "per_image"      the KL summed over the rows of each image and averaged over the images (mean over images, not rows).
"""
import math

import torch

from . import vae as OV

MUTATIONS = ("noisy_logits", "no_centring", "per_image")


def kl_rows(logits):
    """KL_r of every row of logits [..., K] -> [...] (computed with l - lse, never log q)."""
    z = logits - torch.logsumexp(logits, -1, keepdim=True)
    return (z.exp() * z).sum(-1) + math.log(logits.shape[-1])


class _NoCentring(torch.autograd.Function):
    """Value of kl_rows(l).sum(); gradient q (l - lse) without the - e_r term (mutation "no_centring")."""

    @staticmethod
    def forward(ctx, logits):
        ctx.save_for_backward(logits)
        return kl_rows(logits).sum()

    @staticmethod
    def backward(ctx, g):
        (logits,) = ctx.saved_tensors
        z = logits - torch.logsumexp(logits, -1, keepdim=True)
        return g * z.exp() * z


def kl_uniform(logits, mutate=None):
    """Mean over the latent rows (every leading index of logits [..., K]) of KL(softmax(l) || Uniform(K)).
    mutate "per_image": sum over each image's rows (logits [B, h, w, K]), mean over the B images."""
    if mutate == "no_centring":
        return _NoCentring.apply(logits) / logits[..., 0].numel()
    kl = kl_rows(logits)
    if mutate == "per_image":
        return kl.reshape(kl.shape[0], -1).sum(-1).mean()
    return kl.mean()


def forward(p, img, u, convblocks, temperature=1.0, hard=True, bf16=False, stack_factor=1, kl_weight=None,
            mutate=None):
    """oracle.vae.forward with the KL term: returns (loss, recon_mse, kl, recon, logits); loss = recon_mse + kl_weight *
    kl.  kl_weight None: exactly oracle.vae.forward's loss (kl None)."""
    assert mutate is None or mutate in MUTATIONS, mutate
    logits = OV.encoder(p, img, convblocks, bf16, stack_factor)
    y = OV.gumbel_softmax(logits, u, temperature, hard)
    out = OV.decoder(p, y, convblocks, bf16, stack_factor)
    mse = ((img - out) ** 2).mean()                                      # src/vae_tf/layers.py:24-25
    if kl_weight is None:
        return mse, mse, None, out, logits
    src = (logits - torch.log(-torch.log(u))) / temperature if mutate == "noisy_logits" else logits
    kl = kl_uniform(src, mutate if mutate != "noisy_logits" else None)
    return mse + kl_weight * kl, mse, kl, out, logits


def loss_and_grads(p, img, u, convblocks, temperature=1.0, hard=True, bf16=False, kl_weight=None, mutate=None):
    """(loss, recon_mse, kl, recon, logits, grads) with autograd's gradients of the objective."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    loss, mse, kl, out, logits = forward(leaves, img, u, convblocks, temperature, hard, bf16, kl_weight=kl_weight,
                                         mutate=mutate)
    loss.backward()
    return (loss.detach(), mse.detach(), None if kl is None else kl.detach(), out.detach(), logits.detach(),
            {k: v.grad for k, v in leaves.items()})


def kl_grad(logits, c):
    """Closed form of d(c * sum_r KL_r) / d l: c q (l - lse - e), e_r = sum_k q_rk (l_rk - lse_r)."""
    z = logits - torch.logsumexp(logits, -1, keepdim=True)
    q = z.exp()
    return c * q * (z - (q * z).sum(-1, keepdim=True))


def first_max_codes(logits):
    """First-maximum code of every row of logits [..., K]; a row with a NaN gets code 0."""
    flat = logits.reshape(-1, logits.shape[-1])
    nan = torch.isnan(flat).any(-1)
    clean = torch.where(torch.isnan(flat), torch.full_like(flat, -math.inf), flat)
    m = clean.max(-1, keepdim=True).values
    first = (clean == m).to(torch.int64).argmax(-1)        # first index attaining the maximum
    return torch.where(nan, torch.zeros_like(first), first)


def codebook_usage(logits):
    """(counts int64 [K], codes_used, perplexity) of the first-maximum codes of logits [..., K]."""
    K = logits.shape[-1]
    counts = torch.bincount(first_max_codes(logits), minlength=K)
    return (counts,) + usage_of_counts(counts)


def usage_of_counts(counts):
    """(codes_used, perplexity = exp(-sum p log p)) of a code histogram."""
    c = counts.double()
    p = c[c > 0] / c.sum()
    return int((c > 0).sum()), float(torch.exp(-(p * p.log()).sum()))


def kl_weight(step, params):
    """beta_t = kl_loss_weight * min(step / kl_anneal_steps, 1), or kl_loss_weight without the anneal key."""
    beta = params.get("kl_loss_weight")
    if beta is None:
        return None
    n = params.get("kl_anneal_steps")
    return beta * min(step / n, 1.0) if n else beta
