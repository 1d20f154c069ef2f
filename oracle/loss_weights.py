"""ORACLE (test infrastructure, NOT product code) — the weighted DALL-E loss with mtf's z-loss.

The reference's loss is the mean cross-entropy over every position (oracle/dalle.py, src/dalle_mtf/models.py:348-359).
The extension weights text and image rows separately and adds z * lse^2 to every row (mtf's `z_loss` argument of
softmax_cross_entropy_with_logits, pinned to 0 in the reference at models.py:350-351):

    row t of a sequence predicts labels[t];  it is a text row iff t < TL - 1  (TL = text_seq_len), else an image row
    l_t  = lse_t - logit_t[label_t] + z * lse_t^2
    loss = (w_t * sum_text l / (B (TL - 1)) + w_i * sum_image l / (B (IL + 1))) / (w_t + w_i)
    d loss / d logit = a_c ((1 + 2 z lse) softmax - onehot),  a_c the coefficient of the row's class

B is the global batch.  `LossQuirks` holds the two choices a mutation test flips: the class boundary and the factor 2
of the z-loss gradient.  Nothing in the package imports this module.
"""
from dataclasses import dataclass

import torch

from . import dalle as O


@dataclass
class LossQuirks:
    text_rows_offset: int = -1     # text rows are t < text_seq_len + offset (mutation: 0, the boundary at TL)
    z_grad_factor: float = 2.0     # d(z lse^2) / d lse = 2 z lse (mutation: 1)


def text_mask(seq_len, text_seq_len, quirks=None):
    """bool [S]: rows whose target is a text token."""
    q = quirks or LossQuirks()
    return torch.arange(seq_len) < text_seq_len + q.text_rows_offset


def coefficients(weights, text_seq_len, image_seq_len, global_batch, quirks=None):
    """(a_text, a_image) as Python floats (float64).  weights None: 1 / (B S) for every row (the reference)."""
    S = text_seq_len + image_seq_len
    n_text = int(text_mask(S, text_seq_len, quirks).sum())
    n_image = S - n_text
    if weights is None:
        return 1.0 / (global_batch * S), 1.0 / (global_batch * S)
    wt, wi = weights
    a_text = wt / ((wt + wi) * global_batch * n_text) if n_text else 0.0
    return a_text, wi / ((wt + wi) * global_batch * n_image)


def row_coefficients(S, text_seq_len, image_seq_len, weights, global_batch, quirks=None, dtype=torch.float64):
    a_text, a_image = coefficients(weights, text_seq_len, image_seq_len, global_batch, quirks)
    mask = text_mask(S, text_seq_len, quirks)
    return torch.where(mask, torch.tensor(a_text, dtype=dtype), torch.tensor(a_image, dtype=dtype)), mask


def weighted_loss(logits, labels, text_seq_len, image_seq_len, weights, z, global_batch=None, quirks=None):
    """logits [B, S, V] (fp32 or fp64, autograd-friendly), labels [B, S].  Returns (loss, rows, parts): rows = l_t,
    parts = (text-row mean CE, image-row mean CE, mean z-term), every mean over the global batch."""
    B, S, _ = logits.shape
    Bg = B if global_batch is None else global_batch
    lse = torch.logsumexp(logits, -1)
    ce = lse - logits.gather(-1, labels[..., None]).squeeze(-1)
    zt = z * lse * lse
    rows = ce + zt
    a, mask = row_coefficients(S, text_seq_len, image_seq_len, weights, Bg, quirks, dtype=logits.dtype)
    loss = (rows * a).sum()
    n_text = int(mask.sum())
    parts = (ce[:, mask].sum() / (Bg * max(n_text, 1)), ce[:, ~mask].sum() / (Bg * (S - n_text)), zt.sum() / (Bg * S))
    return loss, rows, parts


def dlogits(logits, labels, text_seq_len, image_seq_len, weights, z, global_batch=None, quirks=None):
    """The explicit gradient a_c ((1 + f z lse) softmax - onehot), f = quirks.z_grad_factor, of logits [T, V] whose
    rows are consecutive positions of sequences of length S = TL + IL (float64 recommended)."""
    q = quirks or LossQuirks()
    T, V = logits.shape
    S = text_seq_len + image_seq_len
    Bg = T // S if global_batch is None else global_batch
    a, _ = row_coefficients(S, text_seq_len, image_seq_len, weights, Bg, quirks, dtype=logits.dtype)
    a = a.to(logits.device).repeat(T // S + 1)[:T]
    lse = torch.logsumexp(logits, -1)
    p = torch.exp(logits - lse[:, None])
    onehot = torch.zeros_like(p).scatter_(1, labels.long()[:, None], 1.0)
    return a[:, None] * ((1 + q.z_grad_factor * z * lse)[:, None] * p - onehot)


def loss_and_grads(params, tokens, cfg, weights, z, bf16=False, global_batch=None, quirks=None):
    """oracle.dalle's graph with the weighted loss on top of its logits; gradients by autograd."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    _, _, logits = O.forward(leaves, tokens, cfg, bf16=bf16)
    labels = O.shift_labels(tokens, cfg.eos_token_id)
    loss, rows, parts = weighted_loss(logits, labels, cfg.text_seq_len, cfg.image_seq_len, weights, z, global_batch,
                                      quirks)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), rows.detach(), tuple(p.detach() for p in parts), logits.detach(), grads
