"""A taming-transformers VQGAN (VQModel with its Encoder, VectorQuantizer and Decoder) restated in PyTorch from the
architecture in DESIGN.md §4; taming itself is not needed.  It reads a state dict with taming's key names and shapes
(conv weights OIHW), so one seeded synthetic checkpoint feeds both this oracle and the importer
(dalle_mtf_b200.vqgan_engine.import_taming_state_dict).

Every function computes in the dtype of the state dict it is given: float64 for the tests, bf16 on the GPU (with
channels_last inputs, cuDNN convolutions) for tools/bench_vqgan.py's baseline.  Images are this project's convention,
f32 NHWC in [-1, 1]; codes are [B, h*w] in raster order.

`mut` names a deliberate error (tests/test_vqgan_cpu.py checks that the oracle tests catch each one):
  "pad_before" Downsample pads (1, 0, 1, 0) instead of (0, 1, 0, 1);   "gn_eps" GroupNorm eps 1e-5 instead of 1e-6;
  "no_scale" the attention scores without C^-1/2;                      "softmax_queries" softmax over the queries;
  "relu" ReLU in place of swish;                                       "dec_blocks" num_res_blocks decoder blocks per
  level instead of num_res_blocks + 1;                                 "tie_last" the quantiser's last index on ties.
"""
import math

import torch
import torch.nn.functional as F

MUTANTS = ("pad_before", "gn_eps", "no_scale", "softmax_queries", "relu", "dec_blocks", "tie_last")

# taming's ddconfig of vqgan_imagenet_f16_16384 (num_tokens = its n_embed)
GEOMETRY_F16 = dict(ch=128, ch_mult=[1, 1, 2, 2, 4], num_res_blocks=2, attn_resolutions=[16], z_channels=256,
                    embed_dim=256, num_tokens=16384, resolution=256)
# a small geometry of the same structure: 64 px, a 16 x 16 grid, attention at 16 with C = 128
GEOMETRY_TEST = dict(ch=64, ch_mult=[1, 2, 2], num_res_blocks=1, attn_resolutions=[16], z_channels=64, embed_dim=64,
                     num_tokens=512, resolution=64)


def levels(geo):
    """Per encoder level i: (resolution, width ch * ch_mult[i], attention at that resolution)."""
    res, out = geo["resolution"], []
    for i, m in enumerate(geo["ch_mult"]):
        out.append((res, geo["ch"] * m, res in geo["attn_resolutions"]))
        if i != len(geo["ch_mult"]) - 1:
            res //= 2
    return out


def state_dict_shapes(geo, mut=None):
    """taming key -> shape, in the order VQModel registers its parameters (no loss.* entries)."""
    s = {}
    ch, zc, ed = geo["ch"], geo["z_channels"], geo["embed_dim"]

    def conv(name, cin, cout, k):
        s[name + ".weight"] = (cout, cin, k, k)
        s[name + ".bias"] = (cout,)

    def norm(name, c):
        s[name + ".weight"] = (c,)
        s[name + ".bias"] = (c,)

    def resnet(name, cin, cout):
        norm(name + ".norm1", cin); conv(name + ".conv1", cin, cout, 3)
        norm(name + ".norm2", cout); conv(name + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(name + ".nin_shortcut", cin, cout, 1)

    def attn(name, c):
        norm(name + ".norm", c)
        for p in ("q", "k", "v", "proj_out"):
            conv(f"{name}.{p}", c, c, 1)

    lv = levels(geo)
    conv("encoder.conv_in", 3, ch, 3)
    cin = ch
    for i, (_, w, a) in enumerate(lv):
        for j in range(geo["num_res_blocks"]):
            resnet(f"encoder.down.{i}.block.{j}", cin, w)
            cin = w
            if a:
                attn(f"encoder.down.{i}.attn.{j}", w)
        if i != len(lv) - 1:
            conv(f"encoder.down.{i}.downsample.conv", w, w, 3)
    resnet("encoder.mid.block_1", cin, cin); attn("encoder.mid.attn_1", cin); resnet("encoder.mid.block_2", cin, cin)
    norm("encoder.norm_out", cin); conv("encoder.conv_out", cin, zc, 3)
    conv("decoder.conv_in", zc, lv[-1][1], 3)
    cin = lv[-1][1]
    resnet("decoder.mid.block_1", cin, cin); attn("decoder.mid.attn_1", cin); resnet("decoder.mid.block_2", cin, cin)
    n_dec = geo["num_res_blocks"] + (0 if mut == "dec_blocks" else 1)
    for i in reversed(range(len(lv))):
        _, w, a = lv[i]
        for j in range(n_dec):
            resnet(f"decoder.up.{i}.block.{j}", cin, w)
            cin = w
            if a:
                attn(f"decoder.up.{i}.attn.{j}", w)
        if i != 0:
            conv(f"decoder.up.{i}.upsample.conv", w, w, 3)
    norm("decoder.norm_out", cin); conv("decoder.conv_out", cin, 3, 3)
    conv("quant_conv", zc, ed, 1)
    s["quantize.embedding.weight"] = (geo["num_tokens"], ed)
    conv("post_quant_conv", ed, zc, 1)
    return s


def random_state_dict(geo, seed=0, mut=None):
    """A seeded synthetic checkpoint (f32): conv weights N(0, 1 / fan_in), biases and GroupNorm shifts N(0, 0.1^2),
    GroupNorm scales 1 + N(0, 0.1^2), codebook rows N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in state_dict_shapes(geo, mut).items():
        if k == "quantize.embedding.weight":
            t = torch.randn(shape, generator=g)
        elif len(shape) == 4:
            t = torch.randn(shape, generator=g) / math.sqrt(shape[1] * shape[2] * shape[3])
        elif ".norm" in k and k.endswith(".weight"):
            t = 1 + 0.1 * torch.randn(shape, generator=g)
        else:
            t = 0.1 * torch.randn(shape, generator=g)
        sd[k] = t
    return sd


def _swish(x, mut):
    return F.relu(x) if mut == "relu" else x * torch.sigmoid(x)


def _norm(sd, name, x, mut):
    return F.group_norm(x, 32, sd[name + ".weight"], sd[name + ".bias"], eps=1e-5 if mut == "gn_eps" else 1e-6)


def _conv(sd, name, x, stride=1, padding=None):
    w = sd[name + ".weight"]
    return F.conv2d(x, w, sd[name + ".bias"], stride=stride, padding=w.shape[-1] // 2 if padding is None else padding)


def _resnet(sd, name, x, mut):
    h = _conv(sd, name + ".conv1", _swish(_norm(sd, name + ".norm1", x, mut), mut))
    h = _conv(sd, name + ".conv2", _swish(_norm(sd, name + ".norm2", h, mut), mut))
    if name + ".nin_shortcut.weight" in sd:
        x = _conv(sd, name + ".nin_shortcut", x)
    return x + h


def _attn(sd, name, x, mut):
    B, C, H, W = x.shape
    h = _norm(sd, name + ".norm", x, mut)
    q, k, v = (_conv(sd, f"{name}.{p}", h).reshape(B, C, H * W) for p in ("q", "k", "v"))
    w = torch.bmm(q.transpose(1, 2), k)                      # [B, S queries, S keys]
    if mut != "no_scale":
        w = w * C ** -0.5
    w = torch.softmax(w, dim=1 if mut == "softmax_queries" else 2)
    o = torch.bmm(v, w.transpose(1, 2)).reshape(B, C, H, W)  # o_i = sum_j w_ij v_j
    return x + _conv(sd, name + ".proj_out", o)


def _mid(sd, side, x, mut):
    x = _resnet(sd, f"{side}.mid.block_1", x, mut)
    x = _attn(sd, f"{side}.mid.attn_1", x, mut)
    return _resnet(sd, f"{side}.mid.block_2", x, mut)


def encode_z(sd, geo, img, mut=None):
    """img NHWC [B, H, W, 3] -> quant_conv's output z NHWC [B, h, w, embed_dim]."""
    lv = levels(geo)
    x = _conv(sd, "encoder.conv_in", img.permute(0, 3, 1, 2).to(sd["encoder.conv_in.weight"].dtype))
    for i, (_, _, a) in enumerate(lv):
        for j in range(geo["num_res_blocks"]):
            x = _resnet(sd, f"encoder.down.{i}.block.{j}", x, mut)
            if a:
                x = _attn(sd, f"encoder.down.{i}.attn.{j}", x, mut)
        if i != len(lv) - 1:
            x = F.pad(x, (1, 0, 1, 0) if mut == "pad_before" else (0, 1, 0, 1))
            x = _conv(sd, f"encoder.down.{i}.downsample.conv", x, stride=2, padding=0)
    x = _mid(sd, "encoder", x, mut)
    x = _conv(sd, "encoder.conv_out", _swish(_norm(sd, "encoder.norm_out", x, mut), mut))
    return _conv(sd, "quant_conv", x).permute(0, 2, 3, 1)


def distances(z, codebook):
    """||z_r - e_n||^2 of every latent row z [rows, D] and code e_n."""
    return (z * z).sum(1, keepdim=True) + (codebook * codebook).sum(1)[None, :] - 2 * z @ codebook.T


def nearest_codes(z, codebook, mut=None):
    """argmin_n ||z_r - e_n||^2 with the first index on ties (torch.argmin's rule), int64 [rows]."""
    d = distances(z.reshape(-1, codebook.shape[1]), codebook)
    if mut == "tie_last":
        return d.shape[1] - 1 - torch.argmin(d.flip(1), dim=1)
    return torch.argmin(d, dim=1)


def encode_codes(sd, geo, img, mut=None):
    z = encode_z(sd, geo, img, mut)
    return nearest_codes(z, sd["quantize.embedding.weight"], mut).view(img.shape[0], -1)


def decode(sd, geo, codes, mut=None):
    """codes [B, h*w] -> images NHWC [B, H, W, 3], clamped to [-1, 1]."""
    lv = levels(geo)
    B, n = codes.shape
    hw = int(round(math.sqrt(n)))
    z = sd["quantize.embedding.weight"][codes.reshape(-1).long()].view(B, hw, hw, -1).permute(0, 3, 1, 2)
    x = _conv(sd, "decoder.conv_in", _conv(sd, "post_quant_conv", z))
    x = _mid(sd, "decoder", x, mut)
    n_dec = geo["num_res_blocks"] + (0 if mut == "dec_blocks" else 1)
    for i in reversed(range(len(lv))):
        for j in range(n_dec):
            x = _resnet(sd, f"decoder.up.{i}.block.{j}", x, mut)
            if lv[i][2]:
                x = _attn(sd, f"decoder.up.{i}.attn.{j}", x, mut)
        if i != 0:
            x = _conv(sd, f"decoder.up.{i}.upsample.conv", F.interpolate(x, scale_factor=2.0, mode="nearest"))
    x = _conv(sd, "decoder.conv_out", _swish(_norm(sd, "decoder.norm_out", x, mut), mut))
    return x.clamp(-1, 1).permute(0, 2, 3, 1)


def to(sd, dtype, device="cpu"):
    return {k: v.to(device=device, dtype=dtype) for k, v in sd.items()}
