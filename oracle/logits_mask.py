"""ORACLE (test infrastructure, NOT product code) — the modality logits mask (DALLE-pytorch's logits_mask).

Row t of a sequence of length S = TL + IL predicts labels[t].  It is a text row iff t < TL - 1 (its target is a text
token), else an image row (an image code, or EOS at t = S - 1).  With the mask each row normalises over one window of
the vocabulary:

    text row:   ids [0, image_offset)        image row:   ids [image_offset, V)   (the image codes and EOS)
    l_t  = lse_window_t - logit_t[label_t] + z * lse_window_t^2
    d l_t / d logit = (1 + 2 z lse_window) softmax_window - onehot  inside the window, 0 outside

The means, the text / image weighting and the z-loss are oracle/loss_weights.py's, applied to the logits with -inf
outside each row's window.  `Quirks` holds the two choices a mutation test flips: the class boundary of the windows
(at TL instead of TL - 1) and whether EOS belongs to the image window.  Nothing in the package imports this module.
"""
from dataclasses import dataclass

import torch

from . import dalle as O
from . import loss_weights as OW


@dataclass
class Quirks:
    text_rows_offset: int = -1     # text rows are t < text_seq_len + offset (mutation: 0, the boundary at TL)
    eos_in_image_window: bool = True   # mutation: False, the image window stops before EOS


def window_mask(S, text_seq_len, image_offset, V, quirks=None, device=None):
    """bool [S, V]: True where column v lies inside row t's window."""
    q = quirks or Quirks()
    text = torch.arange(S, device=device) < text_seq_len + q.text_rows_offset
    v = torch.arange(V, device=device)
    image_end = V if q.eos_in_image_window else V - 1
    return torch.where(text[:, None], (v < image_offset)[None, :], ((v >= image_offset) & (v < image_end))[None, :])


def masked_logits(logits, text_seq_len, image_offset, quirks=None):
    """logits [..., S, V] with -inf outside each row's window (differentiable; zero gradient outside)."""
    S, V = logits.shape[-2:]
    m = window_mask(S, text_seq_len, image_offset, V, quirks, logits.device)
    return torch.where(m, logits, torch.tensor(-float("inf"), dtype=logits.dtype, device=logits.device))


def masked_loss(logits, labels, text_seq_len, image_seq_len, image_offset, weights=None, z=0.0, global_batch=None,
                quirks=None):
    """logits [B, S, V], labels [B, S].  (loss, rows, parts) of oracle.loss_weights.weighted_loss on the windowed
    logits; weights None and z 0 is the mean of the rows over the global batch's B S positions."""
    ml = masked_logits(logits, text_seq_len, image_offset, quirks)
    return OW.weighted_loss(ml, labels, text_seq_len, image_seq_len, weights, z, global_batch)


def dlogits(logits, labels, text_seq_len, image_seq_len, image_offset, weights=None, z=0.0, global_batch=None,
            quirks=None):
    """The explicit gradient of masked_loss with respect to logits [T, V] whose rows are consecutive positions of
    sequences of length S = TL + IL: a_c ((1 + 2 z lse_window) softmax_window - onehot), exactly 0 outside the window
    (float64 recommended)."""
    T, V = logits.shape
    S = text_seq_len + image_seq_len
    m = window_mask(S, text_seq_len, image_offset, V, quirks, logits.device)
    m = m.repeat(T // S + 1, 1)[:T]
    ml = torch.where(m, logits, torch.tensor(-float("inf"), dtype=logits.dtype, device=logits.device))
    return OW.dlogits(ml, labels, text_seq_len, image_seq_len, weights, z, global_batch)


def loss_and_grads(params, tokens, cfg, image_offset, weights=None, z=0.0, global_batch=None, quirks=None,
                   forward=None, mask=True):
    """Autograd of masked_loss on top of a forward pass: (loss, rows, parts, logits, grads).  forward(leaves, tokens)
    returns (loss, loss_batch, logits) (default oracle.dalle.forward with cfg); cfg.eos_token_id is the last id.
    mask False: the same with every row over the whole vocabulary (oracle.loss_weights.weighted_loss of the logits)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    fwd = forward or (lambda p, t: O.forward(p, t, cfg))
    _, _, logits = fwd(leaves, tokens)
    labels = O.shift_labels(tokens, logits.shape[-1] - 1)
    if mask:
        loss, rows, parts = masked_loss(logits, labels, cfg.text_seq_len, cfg.image_seq_len, image_offset, weights, z,
                                        global_batch, quirks)
    else:
        loss, rows, parts = OW.weighted_loss(logits, labels, cfg.text_seq_len, cfg.image_seq_len, weights, z,
                                             global_batch)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), rows.detach(), tuple(p.detach() for p in parts), logits.detach(), grads
