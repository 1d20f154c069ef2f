"""ORACLE (test infrastructure, NOT product code) — the discrete VAE's optional logit-Laplace reconstruction loss (an
extension: the reference's objective is MSE; DESIGN.md §4), on top of oracle/vae.py and oracle/vae_kl.py, which it
leaves as they are.

  The decoder's final 1x1 conv has 2 C_p outputs (C_p = C s^2, the packed channels): mu = [0, C_p), ln b = [C_p, 2 C_p),
  both in the packed (space_to_depth) channel order.  oracle.vae.decoder(..., stack_factor=1) returns them packed.
  Target: y = clamp(eps + (1 - 2 eps)(x + 1) / 2, eps, 1 - eps), eps = 0.1, t = logit(y).
  Per subpixel:  nll = ln 2 + ln b + ln y + ln(1 - y) + |t - mu| / b   (a density on (0, 1), Jacobian included).
  Objective: mean nll (+ beta_t KL).  Image-space output: xhat = 2 clamp((sigmoid(mu) - eps) / (1 - 2 eps), 0, 1) - 1;
  recon_mse = mean (xhat - x)^2, a monitor.

Mutation switches (`mutate`), for tests that must tell the engine apart from plausible mistakes:
  "wrong_eps"       targets mapped with eps = 0.05 instead of 0.1;
  "swap_halves"     mu and ln b exchanged;
  "mu_pixel_space"  xhat = mu (no sigmoid, no rescaling);
  "no_jacobian"     nll without ln y + ln(1 - y).
"""
import math

import torch

from . import vae as OV
from . import vae_kl as OK

EPS = 0.1
MUTATIONS = ("wrong_eps", "swap_halves", "mu_pixel_space", "no_jacobian")


def init_params(convblocks, num_tokens, input_channels=3, stack_factor=1, seed=0):
    """oracle.vae.init_params with the final 1x1 conv widened to 2 C_p outputs (glorot_uniform kernel, zero bias)."""
    p = OV.init_params(convblocks, num_tokens, input_channels, stack_factor, seed)
    cin = p["decoder/conv2d/kernel"].shape[2]
    cout = 2 * input_channels * stack_factor ** 2
    g = torch.Generator().manual_seed(seed + 1)
    limit = math.sqrt(6.0 / (cin + cout))
    p["decoder/conv2d/kernel"] = (torch.rand(1, 1, cin, cout, generator=g) * 2 - 1) * limit
    p["decoder/conv2d/bias"] = torch.zeros(cout)
    return p


def target(x, eps=EPS):
    """(y, t): the image x in [-1, 1] mapped into [eps, 1 - eps] and its logit."""
    y = (eps + (1 - 2 * eps) * (x + 1) / 2).clamp(eps, 1 - eps)
    return y, torch.log(y) - torch.log1p(-y)


def split(stats, mutate=None):
    """(mu, ln b) of packed stats [..., 2 C_p]."""
    cp = stats.shape[-1] // 2
    mu, lb = stats[..., :cp], stats[..., cp:]
    return (lb, mu) if mutate == "swap_halves" else (mu, lb)


def nll(stats, x, mutate=None):
    """Per-subpixel logit-Laplace NLL [..., C_p] of the packed target x [..., C_p] under stats [..., 2 C_p]."""
    mu, lb = split(stats, mutate)
    y, t = target(x, 0.05 if mutate == "wrong_eps" else EPS)
    jac = 0 if mutate == "no_jacobian" else torch.log(y) + torch.log1p(-y)
    return math.log(2) + lb + jac + (t - mu).abs() * torch.exp(-lb)


def image(stats, mutate=None):
    """Image-space output [..., C_p] in [-1, 1] of packed stats [..., 2 C_p]."""
    mu, _ = split(stats, mutate)
    if mutate == "mu_pixel_space":
        return mu
    return 2 * ((torch.sigmoid(mu) - EPS) / (1 - 2 * EPS)).clamp(0, 1) - 1


def grads(stats, x, c):
    """Closed forms of d(c * sum nll) / d(mu, ln b): (-c sign(t - mu) / b, c (1 - |t - mu| / b))."""
    mu, lb = split(stats)
    _, t = target(x)
    ib = torch.exp(-lb)
    return -c * torch.sign(t - mu) * ib, c * (1 - (t - mu).abs() * ib)


def density(u, mu, b):
    """The logit-Laplace density at u in (0, 1): exp(-nll) with y = u (for integration checks)."""
    t = math.log(u) - math.log1p(-u)
    return math.exp(-(math.log(2 * b) + math.log(u) + math.log1p(-u) + abs(t - mu) / b))


def forward(p, img, u, convblocks, temperature=1.0, hard=True, bf16=False, stack_factor=1, kl_weight=None,
            mutate=None):
    """Returns (loss, recon_nll, recon_mse, kl, xhat, logits); loss = recon_nll + kl_weight * kl (kl None without
    kl_weight).  xhat is unpacked to the image's layout."""
    assert mutate is None or mutate in MUTATIONS, mutate
    logits = OV.encoder(p, img, convblocks, bf16, stack_factor)
    y = OV.gumbel_softmax(logits, u, temperature, hard)
    stats = OV.decoder(p, y, convblocks, bf16, stack_factor=1)          # packed [N, H/s, W/s, 2 C_p]
    x = OV.space_to_depth(img, stack_factor) if stack_factor > 1 else img
    rec = nll(stats, x, mutate).mean()
    xhat = image(stats, mutate)
    mse = ((xhat - x) ** 2).mean().detach()
    if stack_factor > 1:
        xhat = OV.depth_to_space(xhat, stack_factor)
    if kl_weight is None:
        return rec, rec, mse, None, xhat, logits
    kl = OK.kl_uniform(logits)
    return rec + kl_weight * kl, rec, mse, kl, xhat, logits


def loss_and_grads(p, img, u, convblocks, temperature=1.0, hard=True, bf16=False, stack_factor=1, kl_weight=None,
                   mutate=None):
    """(loss, recon_nll, recon_mse, kl, xhat, logits, grads) with autograd's gradients of the objective."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    loss, rec, mse, kl, xhat, logits = forward(leaves, img, u, convblocks, temperature, hard, bf16, stack_factor,
                                               kl_weight, mutate)
    loss.backward()
    return (loss.detach(), rec.detach(), mse, None if kl is None else kl.detach(), xhat.detach(), logits.detach(),
            {k: v.grad for k, v in leaves.items()})


def decode(p, codes, convblocks, bf16=False, stack_factor=1):
    """Image-space output [N, H, W, C] of the decoder on one-hot codes [N, h, w] (int64)."""
    K = p["codebook/codebook"].shape[1]
    y = torch.nn.functional.one_hot(codes, K).to(torch.float32)
    xhat = image(OV.decoder(p, y, convblocks, bf16, stack_factor=1))
    return OV.depth_to_space(xhat, stack_factor) if stack_factor > 1 else xhat


def beta_from_paper(beta_paper, image_size, channels, grid):
    """kl_loss_weight equivalent to the paper's beta on its per-image ELB: beta h w / (H W C) for a grid x grid code
    grid (the ELB divided by the H W C subpixels is mean nll + beta h w / (H W C) mean KL)."""
    return beta_paper * grid * grid / (image_size * image_size * channels)
