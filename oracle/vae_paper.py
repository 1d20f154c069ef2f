"""ORACLE (test infrastructure, NOT product code) — the DALL-E paper's discrete-VAE network (architecture "dalle_paper",
an extension: the reference's network is oracle/vae.py's).  It restates the dVAE OpenAI published with the paper
(encoder.py / decoder.py of the dall_e package) in this repository's layouts: activations NHWC, kernels HWIO, every
conv SAME with stride 1.  The quantiser and the losses are oracle/vae.py's, oracle/vae_kl.py's and
oracle/vae_logit_laplace.py's, unchanged.

  g(x) = relu(x).  Block(n_in, n_out), h = n_out / 4, gain = 1 / (group_count * n_blk_per_group)^2:
      y = id(x) + gain * res(x),  id = 1x1 conv if n_in != n_out else identity,
      res = conv_4(g(conv_3(g(conv_2(g(conv_1(g(x)))))))),  the gain applying to conv_4's bias too.
      Encoder block kernels 3x3, 3x3, 3x3, 1x1 (n_in -> h -> h -> h -> n_out); decoder block 1x1, 3x3, 3x3, 3x3.
  Encoder: input 7x7 conv C -> n_hid; group k = 1..G of width 2^(k-1) n_hid (its first block reads the previous
      width), every group but the last followed by a 2x2 stride-2 max-pool; output relu then a 1x1 conv (with bias,
      f32) to num_tokens = the logits.
  Decoder: input 1x1 conv (with bias, f32) num_tokens -> n_init of the quantiser's one-hot (its own weights, not the
      encoder's); group k of width 2^(G-k) n_hid, every group but the last followed by a 2x nearest upsample; output
      relu then a 1x1 conv n_hid -> C (MSE) or 2 C (logit-Laplace, mu | ln b).
  Max-pool tie rule: the gradient goes to the FIRST maximum of the window in raster order (0,0), (0,1), (1,0), (1,1).

bf16 policy (bf16=True), the engine's rounding points: the 7x7 input conv is f32 arithmetic on the f32 image and
kernel with its output rounded; every block conv uses its kernel rounded to bf16 (f32 bias, f32 sums) and rounds its
output (conv_1..3 after the ReLU); the block output rounds gain * r + id once, r = conv_4's rounded output and id the
rounded 1x1 output or x; pool / upsample / ReLU are exact; the two projections are f32 (the activations they read are
bf16 values already); the decoder's output conv (f32 kernel, direct kernel) rounds its output.

Mutation switches (`mutate`), for tests that must tell the engine apart from plausible mistakes:
  "gain_one"           blocks without the post-gain (gain 1);
  "tie_last"           max-pool gradient to the LAST maximum of the window;
  "no_preact"          conv_1 reads x instead of relu(x);
  "tied_decoder_input" the decoder input is the one-hot times the transposed encoder output kernel (its first n_init
                       rows), not the decoder's own input conv.
"""
import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

from . import vae as OV
from . import vae_kl as OK
from . import vae_logit_laplace as OL

MUTATIONS = ("gain_one", "tie_last", "no_preact", "tied_decoder_input")


def check_geometry(image_size, n_hid=256, n_blk_per_group=2, group_count=4, n_init=128):
    """Raises ValueError for a geometry the network does not define (image_size not divisible by 2^(G-1), n_hid or
    n_init not a multiple of 8, n_hid < 64, a count < 1)."""
    for k, v in (("n_hid", n_hid), ("n_blk_per_group", n_blk_per_group), ("group_count", group_count),
                 ("n_init", n_init)):
        if isinstance(v, bool) or not isinstance(v, int) or v < 1:
            raise ValueError(f"{k} = {v!r}: must be an integer >= 1")
    if n_hid % 8 or n_hid < 64:
        raise ValueError(f"n_hid = {n_hid}: must be a multiple of 8 and >= 64 (the bottleneck width is width / 4)")
    if n_init % 8:
        raise ValueError(f"n_init = {n_init}: must be a multiple of 8")
    if image_size % (2 ** (group_count - 1)):
        raise ValueError(f"image_size = {image_size} is not divisible by 2^(group_count - 1) = {2 ** (group_count - 1)}")


def grid_size(image_size, group_count=4):
    """Side of the token grid: image_size / 2^(group_count - 1)."""
    return image_size // 2 ** (group_count - 1)


def gain(n_blk_per_group=2, group_count=4):
    return 1.0 / (group_count * n_blk_per_group) ** 2


def _blocks(side, n_hid, n_blk_per_group, group_count, n_init):
    """(prefix, n_in, n_out) of every block of one side, in forward order."""
    out = []
    if side == "encoder":
        prev = n_hid
        widths = [2 ** (k - 1) * n_hid for k in range(1, group_count + 1)]
        kernels = (3, 3, 3, 1)
    else:
        prev = n_init
        widths = [2 ** (group_count - k) * n_hid for k in range(1, group_count + 1)]
        kernels = (1, 3, 3, 3)
    for k, w in enumerate(widths, 1):
        for i in range(1, n_blk_per_group + 1):
            out.append((f"{side}/group_{k}/block_{i}/", prev if i == 1 else w, w, kernels))
        prev = w
    return out


def param_shapes(num_tokens, input_channels=3, n_hid=256, n_blk_per_group=2, group_count=4, n_init=128,
                 logit_laplace=True):
    """OrderedDict name -> shape (HWIO kernels) in the flat layout's order: encoder then decoder, forward order, each
    block's id_path (when n_in != n_out) before its res_path."""
    p = OrderedDict()
    C = input_channels

    def conv(name, k, cin, cout):
        p[name + "/kernel"] = (k, k, cin, cout)
        p[name + "/bias"] = (cout,)

    conv("encoder/input", 7, C, n_hid)
    for side in ("encoder", "decoder"):
        if side == "decoder":
            conv("decoder/input", 1, num_tokens, n_init)
        for pre, n_in, n_out, ks in _blocks(side, n_hid, n_blk_per_group, group_count, n_init):
            h = n_out // 4
            if n_in != n_out:
                conv(pre + "id_path", 1, n_in, n_out)
            chans = (n_in, h, h, h, n_out)
            for j in range(4):
                conv(pre + f"res_path/conv_{j + 1}", ks[j], chans[j], chans[j + 1])
        if side == "encoder":
            conv("encoder/output/conv", 1, 2 ** (group_count - 1) * n_hid, num_tokens)
    conv("decoder/output/conv", 1, n_hid, 2 * C if logit_laplace else C)
    return p


def init_params(num_tokens, input_channels=3, n_hid=256, n_blk_per_group=2, group_count=4, n_init=128,
                logit_laplace=True, seed=0):
    """Normal kernels with std 1 / sqrt(cin kh kw), zero biases (CPU; the engine draws its own on the device)."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    for name, shape in param_shapes(num_tokens, input_channels, n_hid, n_blk_per_group, group_count, n_init,
                                    logit_laplace).items():
        if name.endswith("/bias"):
            p[name] = torch.zeros(shape)
        else:
            p[name] = torch.randn(*shape, generator=g) / math.sqrt(shape[0] * shape[1] * shape[2])
    return p


def _r(x, bf16):
    return x.to(torch.bfloat16).to(torch.float32) if bf16 else x


def max_pool(x, mutate=None):
    """2x2 stride-2 max-pool of NHWC x whose gradient goes to the first maximum of each window in raster order
    (mutation "tie_last": the last)."""
    N, H, W, C = x.shape
    win = x.reshape(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(N, H // 2, W // 2, C, 4)
    if mutate == "tie_last":
        win = win.flip(-1)
    idx = win.argmax(-1, keepdim=True)   # torch.argmax returns the first maximal index
    return win.gather(-1, idx).squeeze(-1)


def upsample(x):
    """2x nearest-neighbour upsampling of NHWC x."""
    return x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)


def _block(p, x, pre, n_in, n_out, ks, g, bf16, mutate):
    W = lambda n: _r(p[n], bf16)
    t = x if mutate == "no_preact" else torch.relu(x)
    for j in range(4):
        nm = pre + f"res_path/conv_{j + 1}"
        t = _r(OV.conv2d_same(t, W(nm + "/kernel"), p[nm + "/bias"], 1), bf16)
        if j < 3:
            t = torch.relu(t)
    idv = _r(OV.conv2d_same(x, W(pre + "id_path/kernel"), p[pre + "id_path/bias"], 1), bf16) if n_in != n_out else x
    return _r(idv + g * t, bf16)


def encoder(p, img, n_hid=256, n_blk_per_group=2, group_count=4, bf16=False, mutate=None):
    """img f32 NHWC in [-1, 1] -> f32 logits [N, h, w, K]."""
    g = 1.0 if mutate == "gain_one" else gain(n_blk_per_group, group_count)
    x = _r(OV.conv2d_same(img, p["encoder/input/kernel"], p["encoder/input/bias"], 1), bf16)
    blocks = _blocks("encoder", n_hid, n_blk_per_group, group_count, None)
    for bi, (pre, n_in, n_out, ks) in enumerate(blocks):
        x = _block(p, x, pre, n_in, n_out, ks, g, bf16, mutate)
        last_in_group = (bi + 1) % n_blk_per_group == 0
        if last_in_group and bi + 1 < len(blocks):
            x = max_pool(x, mutate)
    return OV.conv2d_same(torch.relu(x), p["encoder/output/conv/kernel"], p["encoder/output/conv/bias"], 1)


def decoder(p, y, n_hid=256, n_blk_per_group=2, group_count=4, n_init=128, bf16=False, mutate=None):
    """Quantiser output y f32 [N, h, w, K] -> f32 decoder output [N, H, W, C or 2 C]."""
    g = 1.0 if mutate == "gain_one" else gain(n_blk_per_group, group_count)
    if mutate == "tied_decoder_input":
        w = p["encoder/output/conv/kernel"][0, 0, :n_init, :].t()          # [K, n_init]
        x = y @ w + p["decoder/input/bias"]
    else:
        x = OV.conv2d_same(y, p["decoder/input/kernel"], p["decoder/input/bias"], 1)
    x = _r(x, bf16)
    blocks = _blocks("decoder", n_hid, n_blk_per_group, group_count, n_init)
    for bi, (pre, n_in, n_out, ks) in enumerate(blocks):
        x = _block(p, x, pre, n_in, n_out, ks, g, bf16, mutate)
        if (bi + 1) % n_blk_per_group == 0 and bi + 1 < len(blocks):
            x = upsample(x)
    out = OV.conv2d_same(torch.relu(x), p["decoder/output/conv/kernel"], p["decoder/output/conv/bias"], 1)
    return _r(out, bf16)


def forward(p, img, u, n_hid=256, n_blk_per_group=2, group_count=4, n_init=128, temperature=1.0, hard=True,
            bf16=False, logit_laplace=False, kl_weight=None, mutate=None):
    """Returns (loss, recon_term, recon_mse, kl, out, logits).  recon_term is the MSE (out = the reconstruction) or the
    mean logit-Laplace NLL (out = the image-space output); loss = recon_term + kl_weight * kl (kl None without)."""
    assert mutate is None or mutate in MUTATIONS, mutate
    logits = encoder(p, img, n_hid, n_blk_per_group, group_count, bf16, mutate)
    y = OV.gumbel_softmax(logits, u, temperature, hard)
    stats = decoder(p, y, n_hid, n_blk_per_group, group_count, n_init, bf16, mutate)
    if logit_laplace:
        rec = OL.nll(stats, img).mean()
        out = OL.image(stats)
        mse = ((out - img) ** 2).mean().detach()
    else:
        out = stats
        rec = ((img - out) ** 2).mean()
        mse = rec.detach()
    if kl_weight is None:
        return rec, rec, mse, None, out, logits
    kl = OK.kl_uniform(logits)
    return rec + kl_weight * kl, rec, mse, kl, out, logits


def loss_and_grads(p, img, u, **kw):
    """(loss, recon_term, recon_mse, kl, out, logits, grads) with autograd's gradients of the objective."""
    leaves = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    loss, rec, mse, kl, out, logits = forward(leaves, img, u, **kw)
    loss.backward()
    return (loss.detach(), rec.detach(), mse, None if kl is None else kl.detach(), out.detach(), logits.detach(),
            {k: v.grad for k, v in leaves.items()})


def encode_tokens(p, img, **kw):
    """First-maximum code of every latent row, [B, h * w]."""
    logits = encoder(p, img, **kw)
    return logits.argmax(-1).reshape(img.shape[0], -1)


def decode(p, codes, n_hid=256, n_blk_per_group=2, group_count=4, n_init=128, bf16=False, logit_laplace=False):
    """Decoder output on one-hot codes [N, h, w] (int64): the image-space output (logit-Laplace) or the
    reconstruction (MSE)."""
    K = p["decoder/input/kernel"].shape[2]
    y = F.one_hot(codes, K).to(torch.float32)
    out = decoder(p, y, n_hid, n_blk_per_group, group_count, n_init, bf16)
    return OL.image(out) if logit_laplace else out
