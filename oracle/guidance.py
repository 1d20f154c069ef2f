"""ORACLE (test infrastructure, NOT product code) — classifier-free guidance and caption dropout.

  guided_logits(c, u, s)  the per-op float32 combination u + s * (c - u) that db200_sample_rows_guided applies to a
                          (conditional, unconditional) pair of logit rows before temperature, top-k / top-p
                          (oracle/sampling.py keep_mask) and the Gumbel-max;
  caption_dropped(...)    the caption-dropout decisions of db200_assemble_tokens_ex: the masks of oracle/philox.py at
                          site SITE_CAPTION in the elementwise layout with cols = 1 over sequences, sequence e = row0 + b
                          reading word e & 3 of block e >> 2; its caption is dropped iff that word < floor(rate * 2^32).
Nothing in the package imports this module.
"""
import numpy as np

from .philox import keep_elementwise

SITE_CAPTION = 0xFFFFFFFF


def guided_logits(c, u, s):
    """float32 u + s * (c - u), each op rounded to float32: c the conditional, u the unconditional logits, s the
    guidance scale."""
    c, u = np.asarray(c, dtype=np.float32), np.asarray(u, dtype=np.float32)
    s = np.float32(s)
    with np.errstate(invalid="ignore", over="ignore"):
        return (u + s * (c - u)).astype(np.float32)


def caption_dropped(rate, seed, step, B, row0=0):
    """bool [B]: sequences row0 .. row0 + B - 1 whose caption is replaced by padding at optimiser step `step`."""
    return ~keep_elementwise(rate, seed, step, SITE_CAPTION, B, 1, row0)[:, 0]
