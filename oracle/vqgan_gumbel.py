"""taming-transformers' GumbelVQ (VQModel with GumbelQuantize) restated on top of oracle/vqgan.py, whose encoder and
decoder it reuses unchanged.  A geometry with "quantizer": "gumbel" replaces the codebook quantize.embedding.weight
with GumbelQuantize's quantize.proj (a 1x1 conv z_channels -> n_embed, OIHW weight and bias) and quantize.embed.weight
[n_embed, embed_dim].  The codes are the argmax of the logits z . proj_n + bias_n, the mode of taming's hard
Gumbel-softmax draw (DESIGN.md §4), first index on ties; decoding reads quantize.embed.weight, as DALLE-pytorch's
`one_hot @ quantize.embed.weight` does.

Every function computes in the dtype of the state dict it is given, as oracle/vqgan.py's do.

`mut` names a deliberate error (tests/test_vqgan_gumbel_cpu.py checks that the GPU tests catch each one):
  "gumbel_no_bias" the logits without proj's bias;   "gumbel_decode_proj" decoding through proj's rows instead of
  embed's;                                           "gumbel_tie_last" the last index on tied logits.
oracle/vqgan.py's own mutants apply to the shared encoder and decoder.
"""
import math

import torch

from oracle import vqgan as V

GUMBEL_MUTANTS = ("gumbel_no_bias", "gumbel_decode_proj", "gumbel_tie_last")

# taming's ddconfig of vqgan_gumbel_f8 (8192 codes, a 32 x 32 grid: attention at S = 1024 with C = 512)
GEOMETRY_GUMBEL_F8 = dict(ch=128, ch_mult=[1, 1, 2, 4], num_res_blocks=2, attn_resolutions=[32], z_channels=256,
                          embed_dim=256, num_tokens=8192, resolution=256, quantizer="gumbel")
# a small Gumbel geometry that reaches the same attention: 64 px, a 32 x 32 grid, S = 1024 and C = 512 at level 1 and
# in the mid blocks
GEOMETRY_GUMBEL_TEST = dict(ch=128, ch_mult=[1, 4], num_res_blocks=1, attn_resolutions=[32], z_channels=64,
                            embed_dim=64, num_tokens=512, resolution=64, quantizer="gumbel")


def is_gumbel(geo):
    return geo.get("quantizer", "vq") == "gumbel"


def state_dict_shapes(geo, mut=None):
    """taming key -> shape of a GumbelVQ, in oracle/vqgan.py's order with the quantiser's entries in the codebook's
    place: quantize.proj.weight [n_embed, z_channels, 1, 1], quantize.proj.bias, quantize.embed.weight."""
    s = {}
    for k, shape in V.state_dict_shapes(geo, mut).items():
        if k == "quantize.embedding.weight":
            s["quantize.proj.weight"] = (geo["num_tokens"], geo["z_channels"], 1, 1)
            s["quantize.proj.bias"] = (geo["num_tokens"],)
            s["quantize.embed.weight"] = shape
        else:
            s[k] = shape
    return s


def random_state_dict(geo, seed=0, mut=None):
    """A seeded synthetic GumbelVQ checkpoint (f32) with oracle/vqgan.py's distributions: conv weights (proj's too)
    N(0, 1 / fan_in), biases and GroupNorm shifts N(0, 0.1^2), GroupNorm scales 1 + N(0, 0.1^2), embed rows N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in state_dict_shapes(geo, mut).items():
        if k == "quantize.embed.weight":
            t = torch.randn(shape, generator=g)
        elif len(shape) == 4:
            t = torch.randn(shape, generator=g) / math.sqrt(shape[1] * shape[2] * shape[3])
        elif ".norm" in k and k.endswith(".weight"):
            t = 1 + 0.1 * torch.randn(shape, generator=g)
        else:
            t = 0.1 * torch.randn(shape, generator=g)
        sd[k] = t
    return sd


def logits(sd, z, mut=None):
    """GumbelQuantize's logits proj(z) of latent rows z [rows, D]: [rows, num_tokens]."""
    w = sd["quantize.proj.weight"][:, :, 0, 0]
    out = z.reshape(-1, w.shape[1]) @ w.T
    return out if mut == "gumbel_no_bias" else out + sd["quantize.proj.bias"]


def codes(sd, z, mut=None):
    """The mode of taming's hard Gumbel-softmax draw: argmax of the logits, first index on ties, int64 [rows]."""
    lg = logits(sd, z, mut)
    if mut == "gumbel_tie_last":
        return lg.shape[1] - 1 - torch.argmax(lg.flip(1), dim=1)
    return torch.argmax(lg, dim=1)


def encode_codes(sd, geo, img, mut=None):
    """img NHWC [B, H, W, 3] -> codes [B, h*w] (oracle/vqgan.py's encoder and quant_conv, then the logits' argmax)."""
    return codes(sd, V.encode_z(sd, geo, img, mut), mut).view(img.shape[0], -1)


def decode(sd, geo, ids, mut=None):
    """codes [B, h*w] -> images NHWC [B, H, W, 3], clamped to [-1, 1]: embed's rows through oracle/vqgan.py's
    decoder."""
    table = sd["quantize.proj.weight"][:, :, 0, 0] if mut == "gumbel_decode_proj" else sd["quantize.embed.weight"]
    return V.decode({**sd, "quantize.embedding.weight": table}, geo, ids, mut)
