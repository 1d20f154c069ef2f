"""ORACLE (test infrastructure, NOT product code) — the DALL-E paper's input embedding.

The reference embeds positions with one learned vector per position (wpe [S, d], src/dalle_mtf/models.py:203-219)
and pads every caption with one id.  The DALL-E paper (Ramesh et al. 2021, appendix, embedding scheme) instead
  * sums each image token's embedding with a row embedding and a column embedding of the W x W token grid, and
  * pads captions with a separate padding token for each text position.
This module restates both on top of oracle/dalle.py (unchanged) and the forwards that build on it:

  compose_positions(params, cfg)   the [S, d] position table: wpe [TL, d] for the text positions, then
                                   image_row[r] + image_col[c] at TL + r W + c.  With bf16 the sum is of the bf16
                                   parameters and is rounded to bf16 once (the engine's table).
  map_pads(text, ...)              caption ids -> tokens of the text positions: padding_id at position p (and every
                                   position of a dropped caption, oracle/guidance.py) becomes text_vocab_size + p.
  assemble(text, image, ...)       the whole token row; image code i is token image_offset + i.
  forward / loss_and_grads         oracle.dalle_local.forward (which is oracle.dalle / oracle.dalle_dropout when every
                                   layer is global) over the composed table, or any forward of that signature.

With both keys off every function computes, operation for operation, what the forward it wraps computes
(tests/test_paper_embedding_cpu.py).

Mutation switches (`mutate`), for tests that must tell the engine apart from plausible mistakes:
  "transpose"     row and column exchanged (image_row[c] + image_col[r]);
  "pad_plus_one"  pads mapped to text_vocab_size + p + 1;
  "shift_origin"  the grid starts one position late (image token k gets the embedding of k - 1, the first the text
                  table's last row).
Nothing in the package imports this module.
"""
import dataclasses
import math
from dataclasses import dataclass

import torch

from . import dalle_local
from .dalle import _r
from .guidance import caption_dropped

MUTATIONS = ("transpose", "pad_plus_one", "shift_origin")


@dataclass
class InputConfig:
    image_position_embedding: str = "absolute"   # or "row_col"
    per_position_padding: bool = False
    padding_id: int = None


def grid_side(cfg):
    W = math.isqrt(cfg.image_seq_len)
    assert W * W == cfg.image_seq_len, "row / column positions need a square image-token grid"
    return W


def vocab(cfg, inp: InputConfig):
    """(image_offset, V): the first image token id and the vocabulary size with EOS."""
    off = cfg.text_vocab_size + (cfg.text_seq_len if inp.per_position_padding else 0)
    return off, off + cfg.image_vocab_size + 1


def init_params(cfg, inp: InputConfig, seed=0):
    """oracle.dalle.init_params of the model's vocabulary; with row / column positions wpe [TL, d], image_row and
    image_col [W, d] are drawn N(0, 0.01) (models.py:204-208's initialiser) from a second stream seeded seed + 1."""
    from . import dalle as O
    p = O.init_params(_model_cfg(cfg, inp), seed)
    if inp.image_position_embedding == "row_col":
        g = torch.Generator().manual_seed(seed + 1)
        d, W = cfg.n_embd, grid_side(cfg)
        p["positional_embedding/wpe"] = torch.randn(cfg.text_seq_len, d, generator=g) * 0.01
        p["positional_embedding/image_row"] = torch.randn(W, d, generator=g) * 0.01
        p["positional_embedding/image_col"] = torch.randn(W, d, generator=g) * 0.01
    return p


def compose_positions(params, cfg, bf16=False, mutate=None):
    """The [S, d] position table of row / column positions (differentiable in wpe, image_row and image_col)."""
    TL, W = cfg.text_seq_len, grid_side(cfg)
    wpe = _r(params["positional_embedding/wpe"], bf16)
    row = _r(params["positional_embedding/image_row"], bf16)
    col = _r(params["positional_embedding/image_col"], bf16)
    r = torch.arange(W).repeat_interleave(W)      # image token k = r W + c
    c = torch.arange(W).repeat(W)
    if mutate == "transpose":
        r, c = c, r
    img = _r(row[r] + col[c], bf16)
    table = torch.cat([wpe, img], dim=0)
    if mutate == "shift_origin":
        table = torch.cat([table[:TL], table[TL - 1:TL + W * W - 1]], dim=0)
    return table


def map_pads(text, cfg, inp: InputConfig, dropped=None, mutate=None):
    """Tokens of the text positions, int64 [B, TL]: with per-position padding, padding_id at position p (every
    position of a row with dropped[b]) becomes text_vocab_size + p (+ 1 under "pad_plus_one"); without it a dropped
    row is padding_id everywhere (db200_assemble_tokens_ex) and other ids pass through."""
    text = torch.as_tensor(text).long()
    B, TL = text.shape
    drop = torch.zeros(B, dtype=torch.bool) if dropped is None else torch.as_tensor(dropped, dtype=torch.bool)
    if not inp.per_position_padding:
        return torch.where(drop[:, None], torch.full_like(text, inp.padding_id if inp.padding_id is not None else 0),
                           text)
    pads = cfg.text_vocab_size + torch.arange(TL) + (1 if mutate == "pad_plus_one" else 0)
    is_pad = (text == inp.padding_id) | drop[:, None]
    return torch.where(is_pad, pads[None, :].expand(B, TL), text)


def assemble(text, image, cfg, inp: InputConfig, caption_drop=None, mutate=None):
    """The token rows the engine trains on: map_pads(text) then image code i as image_offset + i.  caption_drop:
    (rate, seed, step, row0) of caption dropout (oracle/guidance.py), or None."""
    dropped = None
    if caption_drop is not None:
        rate, seed, step, row0 = caption_drop
        dropped = torch.from_numpy(caption_dropped(rate, seed, step, len(text), row0))
    off, _ = vocab(cfg, inp)
    return torch.cat([map_pads(text, cfg, inp, dropped, mutate), torch.as_tensor(image).long() + off], dim=1)


def _model_cfg(cfg, inp):
    """The base oracles' config of the model's vocabulary (their total_tokens / eos_token_id follow it)."""
    off, _ = vocab(cfg, inp)
    return dataclasses.replace(cfg, text_vocab_size=off)


def forward(params, tokens, cfg, inp: InputConfig, dropout=None, bf16=False, quirks=None, mutate=None, base=None):
    """(loss, loss_batch, logits) of the model with this input embedding.  base: the forward to run (default
    oracle.dalle_local.forward, signature (params, tokens, cfg, dropout, bf16=, quirks=)); cfg carries the attention
    types that forward reads."""
    base = base or dalle_local.forward
    p = dict(params)
    if inp.image_position_embedding == "row_col":
        p["positional_embedding/wpe"] = compose_positions(params, cfg, bf16, mutate)
    elif mutate in ("transpose", "shift_origin"):
        raise ValueError(f"mutation {mutate!r} needs row / column positions")
    return base(p, tokens, _model_cfg(cfg, inp), dropout, bf16=bf16, quirks=quirks)


def loss_and_grads(params, tokens, cfg, inp: InputConfig, dropout=None, bf16=False, quirks=None, mutate=None,
                   base=None):
    """Autograd of forward(): (loss, loss_batch, logits, grads), grads keyed like params (image_row / image_col
    receive the row / column sums of the composed table's gradient)."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, loss_batch, logits = forward(leaves, tokens, cfg, inp, dropout, bf16, quirks, mutate, base)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return loss.detach(), loss_batch.detach(), logits.detach(), grads
