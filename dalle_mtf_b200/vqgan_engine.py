"""A pretrained taming-transformers VQGAN as a frozen image tokenizer (architecture "vqgan"; DESIGN.md §4 holds the
definition and the precision policy, oracle/vqgan.py restates it in PyTorch).  Forward only: encode_tokens for DALL-E
training and decode_tokens for generation.

Parameter names are taming's state-dict keys with "." -> "/" (encoder/down/0/block/0/conv1/weight, ...): conv kernels
HWIO, GroupNorm weights and biases [C], the codebook quantize/embedding/weight [num_tokens, embed_dim] or, for a
Gumbel quantiser ("quantizer": "gumbel", taming's GumbelVQ), quantize/proj/weight [1, 1, embed_dim, num_tokens],
quantize/proj/bias [num_tokens] and quantize/embed/weight [num_tokens, embed_dim].
import_taming_state_dict converts a taming state dict into these names; tools/import_vqgan.py writes the result as a
checkpoint.

Kernels: the 3x3 / 1x1 convolutions on K11 (the wgmma implicit GEMM where the shape qualifies, Cin % 64 == 0; the
3 -> ch input conv and the ch -> 3 output conv on the direct kernel), GroupNorm (+ swish), the AttnBlock's attention,
the codebook gather and the output clamp on K14 (attention over S > 256 positions at C = 512 on its wgmma kernel,
csrc/vqgan_attn.cu), the attention's q|k|v and proj_out 1x1 convs on the GEMM (q, k and v fused into one [C, 3C]
product), nearest 2x upsampling on K11p.  Activations are bf16; quant_conv, the nearest-code
search (or the Gumbel logits) and post_quant_conv run on bf16 hi + lo split operands (fp32-accurate).
"""
import math

import torch

from . import lib as L
from . import ops
from .dalle_engine import ParamLayout
from .vae_engine import BF16, F32, I32, DECODE_PASS_BYTES

GROUPS, EPS = 32, 1e-6
ATTN_MAX_S, ATTN_MAX_C = 256, 512        # db200_attn_noncausal_fwd's range
ATTN_LONG_MAX_S, ATTN_LONG_C = 4096, 512  # db200_attn_noncausal_long_fwd's: ATTN_MAX_S < S <= 4096 at C == 512 only
QUANTIZERS = ("vq", "gumbel")


def attention_in_range(S, C):
    """Whether an AttnBlock over S positions of C channels runs on a kernel: db200_attn_noncausal_fwd for S <= 256
    with C <= 512, db200_attn_noncausal_long_fwd for 256 < S <= 4096 at C == 512 (S a multiple of 64 for both)."""
    if S % 64:
        return False
    return (S <= ATTN_MAX_S and C <= ATTN_MAX_C) or (ATTN_MAX_S < S <= ATTN_LONG_MAX_S and C == ATTN_LONG_C)


def _int(k, v, lo=1):
    if isinstance(v, bool) or not isinstance(v, int) or v < lo:
        raise ValueError(f"{k} = {v!r}: must be an integer >= {lo}")


def check_vqgan_geometry(image_size, ch, ch_mult, num_res_blocks, attn_resolutions, z_channels, embed_dim,
                         num_tokens=None, resolution=None, quantizer="vq"):
    """Raises ValueError, naming the key, for a geometry the kernels do not cover."""
    if quantizer not in QUANTIZERS:
        raise ValueError(f"quantizer = {quantizer!r}: must be one of {QUANTIZERS} (or absent for \"vq\")")
    if quantizer == "gumbel" and embed_dim != z_channels:
        raise ValueError(f"embed_dim = {embed_dim}: a Gumbel quantiser needs embed_dim == z_channels = {z_channels} "
                         "(taming builds its proj on z_channels inputs and applies it to quant_conv's embed_dim outputs)")
    _int("image_size", image_size)
    _int("ch", ch)
    _int("num_res_blocks", num_res_blocks)
    for k, v in (("z_channels", z_channels), ("embed_dim", embed_dim)):
        _int(k, v)
        if v % 64:
            raise ValueError(f"{k} = {v}: must be a multiple of 64 (the wgmma products and split GEMMs)")
    if ch % 64:
        raise ValueError(f"ch = {ch}: must be a multiple of 64 (the wgmma convolutions need Cin % 64 == 0)")
    if not isinstance(ch_mult, (list, tuple)) or not ch_mult:
        raise ValueError(f"ch_mult = {ch_mult!r}: must be a non-empty list of integers")
    for m in ch_mult:
        _int("ch_mult", m)
    if ch * max(ch_mult) > 2048:
        raise ValueError(f"ch * max(ch_mult) = {ch * max(ch_mult)}: GroupNorm covers at most 2048 channels")
    if resolution is not None and resolution != image_size:
        raise ValueError(f"resolution = {resolution}: must equal dataset.image_size = {image_size}")
    if image_size % 2 ** (len(ch_mult) - 1):
        raise ValueError(f"image_size = {image_size} is not divisible by 2^(len(ch_mult) - 1) = "
                         f"{2 ** (len(ch_mult) - 1)}")
    if not isinstance(attn_resolutions, (list, tuple)):
        raise ValueError(f"attn_resolutions = {attn_resolutions!r}: must be a list of integers")
    res = image_size
    for i, m in enumerate(ch_mult):
        if res in attn_resolutions or (i == len(ch_mult) - 1):   # the mid blocks attend at the last resolution
            C, S = ch * m, res * res
            if not attention_in_range(S, C):
                what = "attn_resolutions" if res in attn_resolutions else "image_size / ch_mult (the mid AttnBlock)"
                raise ValueError(f"{what}: attention at {res} x {res} with {C} channels is outside the kernels' range "
                                 f"(S = res^2 a multiple of 64: up to {ATTN_MAX_S} with C up to {ATTN_MAX_C}, or up "
                                 f"to {ATTN_LONG_MAX_S} with C = {ATTN_LONG_C})")
        res //= 2
    if num_tokens is not None:
        _int("num_tokens", num_tokens)


def _levels(geo):
    """Per level i: (resolution, width ch * ch_mult[i], attention at that resolution)."""
    res, out = geo["resolution"], []
    for i, m in enumerate(geo["ch_mult"]):
        out.append((res, geo["ch"] * m, res in geo["attn_resolutions"]))
        if i != len(geo["ch_mult"]) - 1:
            res //= 2
    return out


def network(geo):
    """(encoder steps, decoder steps, ParamLayout) of a geometry.  A step is ("res", name, res, cin, cout),
    ("attn", name, res, C), ("down", name, res, C) or ("up", name, res, C), res its input resolution; the layout holds
    every variable under its taming name with "." -> "/", conv kernels HWIO."""
    lv, nb, hw = _levels(geo), geo["num_res_blocks"], _levels(geo)[-1][0]
    mid = lambda side, C: [("res", f"{side}/mid/block_1", hw, C, C), ("attn", f"{side}/mid/attn_1", hw, C),
                           ("res", f"{side}/mid/block_2", hw, C, C)]
    enc, cin = [], geo["ch"]
    for i, (res, w, a) in enumerate(lv):
        for j in range(nb):
            enc.append(("res", f"encoder/down/{i}/block/{j}", res, cin, w)); cin = w
            if a:
                enc.append(("attn", f"encoder/down/{i}/attn/{j}", res, w))
        if i != len(lv) - 1:
            enc.append(("down", f"encoder/down/{i}/downsample/conv", res, w))
    enc += mid("encoder", cin)
    dec, cin = mid("decoder", lv[-1][1]), lv[-1][1]
    for i in reversed(range(len(lv))):
        res, w, a = lv[i]
        for j in range(nb + 1):
            dec.append(("res", f"decoder/up/{i}/block/{j}", res, cin, w)); cin = w
            if a:
                dec.append(("attn", f"decoder/up/{i}/attn/{j}", res, w))
        if i != 0:
            dec.append(("up", f"decoder/up/{i}/upsample/conv", res, w))

    lay = ParamLayout()
    conv = lambda name, k, ci, co: (lay.add(name + "/weight", (k, k, ci, co)), lay.add(name + "/bias", (co,)))
    norm = lambda name, c: (lay.add(name + "/weight", (c,)), lay.add(name + "/bias", (c,)))

    def steps(lst):
        for s in lst:
            if s[0] == "res":
                name, ci, co = s[1], s[3], s[4]
                norm(name + "/norm1", ci); conv(name + "/conv1", 3, ci, co)
                norm(name + "/norm2", co); conv(name + "/conv2", 3, co, co)
                if ci != co:
                    conv(name + "/nin_shortcut", 1, ci, co)
            elif s[0] == "attn":
                norm(s[1] + "/norm", s[3])
                for p in ("q", "k", "v", "proj_out"):
                    conv(f"{s[1]}/{p}", 1, s[3], s[3])
            else:
                conv(s[1], 3, s[3], s[3])

    zc, ed = geo["z_channels"], geo["embed_dim"]
    conv("encoder/conv_in", 3, 3, geo["ch"]); steps(enc)
    norm("encoder/norm_out", lv[-1][1]); conv("encoder/conv_out", 3, lv[-1][1], zc)
    conv("decoder/conv_in", 3, zc, lv[-1][1]); steps(dec)
    norm("decoder/norm_out", cin); conv("decoder/conv_out", 3, cin, 3)
    conv("quant_conv", 1, zc, ed)
    if geo.get("quantizer", "vq") == "gumbel":
        conv("quantize/proj", 1, ed, geo["num_tokens"])
        lay.add("quantize/embed/weight", (geo["num_tokens"], ed))
    else:
        lay.add("quantize/embedding/weight", (geo["num_tokens"], ed))
    conv("post_quant_conv", 1, ed, zc)
    return enc, dec, lay


# ------------------------------------------------------------------------------------------------------ import
def import_taming_state_dict(sd, geo):
    """taming VQModel state dict (OIHW conv weights) -> this project's named tensors (f32, HWIO kernels).

    geo: {ch, ch_mult, num_res_blocks, attn_resolutions, z_channels, embed_dim, num_tokens, resolution} and optionally
    quantizer ("vq", the default: a VectorQuantizer VQModel; "gumbel": a GumbelVQ).  taming's loss.* entries (LPIPS,
    discriminator) are ignored.  Raises ValueError naming the variable for a checkpoint of the other quantiser, a
    double_z checkpoint and a missing, extra or wrongly shaped tensor."""
    sd = {k: v for k, v in sd.items() if not k.startswith("loss.")}
    if geo.get("quantizer", "vq") == "gumbel":
        if "quantize.embedding.weight" in sd:
            raise ValueError("quantize.embedding.weight: a VectorQuantizer checkpoint (VQModel); set "
                             "\"quantizer\": \"vq\" (or leave it out) in the VAE config")
    else:
        gumbel = [k for k in sd if k == "quantize.embed.weight" or k.startswith("quantize.proj")]
        if gumbel:
            raise ValueError(f"{gumbel[0]}: a Gumbel-quantised checkpoint (GumbelVQ); set \"quantizer\": \"gumbel\" "
                             "in the VAE config")
    w = sd.get("encoder.conv_out.weight")
    if w is not None and w.shape[0] == 2 * geo["z_channels"]:
        raise ValueError(f"encoder.conv_out.weight has {w.shape[0]} = 2 * z_channels outputs: a double_z encoder, "
                         "which a VQGAN does not use")
    lay = network(geo)[2]
    want = {}
    for name in lay.order:   # taming's shapes: conv weights OIHW
        shape = lay.entries[name][1]
        want[name.replace("/", ".")] = (shape[3], shape[2], shape[0], shape[1]) if len(shape) == 4 else shape
    for k in want:
        if k not in sd:
            raise ValueError(f"{k}: missing from the checkpoint (expected shape {want[k]})")
    for k in sd:
        if k not in want:
            raise ValueError(f"{k}: not a tensor of the configured VQGAN geometry")
    out = {}
    for k, shape in want.items():
        t = sd[k]
        if tuple(t.shape) != tuple(shape):
            raise ValueError(f"{k}: shape {tuple(t.shape)}, the configured geometry has {tuple(shape)}")
        t = t.detach().to(torch.float32)
        if t.dim() == 4:
            t = t.permute(2, 3, 1, 0)         # OIHW -> HWIO
        out[k.replace(".", "/")] = t.contiguous()
    return out


def load_taming_checkpoint(path):
    """The state dict of a taming checkpoint: a Lightning .ckpt (its "state_dict") or a bare state dict.  Read with
    weights_only=True, since this is a foreign pickle."""
    try:
        obj = torch.load(path, map_location="cpu", weights_only=True)
    except Exception as e:
        raise ValueError(
            f"{path}: cannot be read with torch.load(weights_only=True) ({type(e).__name__}: {e}).  If you trust the "
            "file, extract its weights once with: python -c \"import torch; "
            f"torch.save(torch.load('{path}', map_location='cpu', weights_only=False)['state_dict'], "
            "'state_dict.pt')\" and import state_dict.pt instead") from None
    if isinstance(obj, dict) and isinstance(obj.get("state_dict"), dict):
        obj = obj["state_dict"]
    if not isinstance(obj, dict) or not all(torch.is_tensor(v) for v in obj.values()):
        raise ValueError(f"{path}: neither a Lightning checkpoint with a state_dict nor a state dict of tensors")
    return obj


# ------------------------------------------------------------------------------------------------------ engine
class VqganEngine:
    def __init__(self, num_tokens, image_size, ch, ch_mult, num_res_blocks, attn_resolutions, z_channels, embed_dim,
                 resolution=None, input_channels=3, device="cuda", quantizer="vq"):
        L.require_device()
        check_vqgan_geometry(image_size, ch, ch_mult, num_res_blocks, attn_resolutions, z_channels, embed_dim,
                             num_tokens, resolution, quantizer)
        if input_channels != 3:
            raise ValueError(f"input_channels = {input_channels}: a VQGAN reads RGB images (3 channels)")
        self.geo = dict(ch=ch, ch_mult=list(ch_mult), num_res_blocks=num_res_blocks,
                        attn_resolutions=list(attn_resolutions), z_channels=z_channels, embed_dim=embed_dim,
                        num_tokens=num_tokens, resolution=image_size, quantizer=quantizer)
        self.gumbel = quantizer == "gumbel"
        # the table decode_tokens gathers codes from: taming's codebook, or GumbelQuantize's embed
        self.codebook = "quantize/embed/weight" if self.gumbel else "quantize/embedding/weight"
        self.K = int(num_tokens)
        self.img_H = self.img_W = self.H = self.W = int(image_size)
        self.img_C = 3
        self.hw = image_size // 2 ** (len(ch_mult) - 1)
        self.image_seq_len = self.hw * self.hw
        self.zc, self.ed = z_channels, embed_dim
        self.device = torch.device(device)
        self.stack_factor = 1

        self.enc, self.dec, self.layout = network(self.geo)
        lay = self.layout
        self.enc_top, self.dec_out_cin = ch * ch_mult[-1], ch * ch_mult[0]
        dev = self.device
        n = lay.size
        self.master = torch.zeros(n, dtype=F32, device=dev)
        self.shadow = torch.zeros(n, dtype=BF16, device=dev)      # bf16 kernels of the wgmma convolutions and GEMMs
        e = lambda *shape, dtype=BF16: torch.zeros(*shape, dtype=dtype, device=dev)
        self.qkv_w = {s[1]: e(s[3], 3 * s[3]) for s in self.enc + self.dec if s[0] == "attn"}     # fused q|k|v [C, 3C]
        self.qkv_b = {s[1]: e(3 * s[3], dtype=F32) for s in self.enc + self.dec if s[0] == "attn"}
        self.qc_hi, self.qc_lo = e(self.zc, self.ed), e(self.zc, self.ed)                       # quant_conv [zc, ed]
        self.pq_hi, self.pq_lo = e(self.ed, self.zc), e(self.ed, self.zc)                       # post_quant_conv
        self.cb_hi, self.cb_lo = e(self.K, self.ed), e(self.K, self.ed)     # codebook, or Gumbel proj^T [K, ed]
        self.cb_bias = e(self.K, dtype=F32)                                 # -||e_n||^2 / 2, or the proj bias
        self._B = None
        self._views = {}
        self._descs = {}

    # -------------------------------------------------------------------------------------------------- parameters
    def _view(self, buf, name):
        key = (buf.data_ptr(), name)
        v = self._views.get(key)
        if v is None:
            v = self._views[key] = self.layout.view(buf, name)
        return v

    def P(self, name):
        return self._view(self.master, name)

    def W16(self, name):
        return self._view(self.shadow, name)

    def n_params(self):
        return sum(math.prod(shape) for _, shape in self.layout.entries.values())

    def load_params(self, named):
        """Named f32 tensors (import_taming_state_dict's names and shapes; extra names are refused)."""
        extra = sorted(set(named) - set(self.layout.order))
        if extra:
            raise L.DB200Error(f"load_params: {extra[0]} is not a variable of this VQGAN")
        for name in self.layout.order:
            if name not in named:
                raise L.DB200Error(f"load_params: {name} missing")
            dst = self.P(name)
            t = named[name]
            if tuple(t.shape) != tuple(dst.shape):
                raise L.DB200Error(f"load_params: {name}: expected {tuple(dst.shape)}, got {tuple(t.shape)}")
            dst.copy_(t.to(device=self.device, dtype=F32))
        self._refresh()

    def export_params(self, source=None):
        flat = self.master if source is None else source
        return {n: self.layout.view(flat, n).detach().float().cpu().clone() for n in self.layout.order}

    def init_params(self, seed=0):
        """Synthetic weights drawn on the device (throughput runs without a checkpoint): conv kernels N(0, 1 / fan_in),
        GroupNorm scales 1, biases 0, codebook (Gumbel embed) rows N(0, 1)."""
        g = torch.Generator(device=self.device).manual_seed(seed)
        self.master.zero_()
        for name in self.layout.order:
            shape = self.layout.entries[name][1]
            if len(shape) == 4:
                self.P(name).copy_(torch.randn(shape, generator=g, device=self.device) / math.sqrt(math.prod(shape[:3])))
            elif name == self.codebook:
                self.P(name).copy_(torch.randn(shape, generator=g, device=self.device))
            elif "/norm" in name and name.endswith("/weight"):
                self.P(name).fill_(1.0)
        self._refresh()

    def _refresh(self):
        """The compute copies of the weights: bf16 kernels, the fused q|k|v products, the split 1x1 convs and the code
        scores' split operand and bias: the codebook with -||e_n||^2 / 2 (summed once here, in float64 on the host), or
        for a Gumbel quantiser proj's kernel transposed to [K, embed_dim] with proj's bias."""
        ops.cast_f32_to_bf16(self.master, self.shadow)
        for name, w in self.qkv_w.items():
            C = w.shape[0]
            for i, p in enumerate(("q", "k", "v")):
                w[:, i * C:(i + 1) * C].copy_(self.W16(f"{name}/{p}/weight").view(C, C))
                self.qkv_b[name][i * C:(i + 1) * C].copy_(self.P(f"{name}/{p}/bias"))
        ops.split_f32(self.P("quant_conv/weight").view(self.zc, self.ed), self.qc_hi, self.qc_lo)
        ops.split_f32(self.P("post_quant_conv/weight").view(self.ed, self.zc), self.pq_hi, self.pq_lo)
        if self.gumbel:
            ops.split_f32(self.P("quantize/proj/weight").view(self.ed, self.K).t().contiguous(), self.cb_hi, self.cb_lo)
            self.cb_bias.copy_(self.P("quantize/proj/bias"))
            return
        cb = self.P("quantize/embedding/weight")
        ops.split_f32(cb, self.cb_hi, self.cb_lo)
        self.cb_bias.copy_((-0.5 * (cb.detach().cpu().double() ** 2).sum(1)).float())

    # -------------------------------------------------------------------------------------------------- buffers
    def _shapes(self):
        """(res, C) of every activation the network holds, with the buffers of each that are alive at once."""
        shapes = {}

        def need(res, C, n):
            shapes[(res, C)] = max(shapes.get((res, C), 0), n)
        need(self.H, self.geo["ch"], 1)                    # encoder/conv_in's output
        # encoder/norm_out (x, t) and conv_out's output h, which must not be t; decoder/conv_in's input (the cast of
        # post_quant_conv) and its output.  With z_channels == ch * ch_mult[-1] all of them share one pool.
        if self.zc == self.enc_top:
            need(self.hw, self.zc, 2)
        else:
            need(self.hw, self.zc, 1)
            need(self.hw, self.enc_top, 2)
        need(self.H, self.dec_out_cin, 2)                  # decoder/norm_out (x, t)
        for steps in (self.enc, self.dec):
            for s in steps:
                if s[0] == "res":    # x, t = GN1(x) | h = conv1(t), t = GN2(h), shortcut s, out
                    need(s[2], s[3], 2)
                    need(s[2], s[4], 3)
                elif s[0] == "attn":  # x, t = GN(x), out
                    need(s[2], s[3], 3)
                elif s[0] == "down":
                    need(s[2] // 2, s[3], 1)
                else:                 # upsampled, conv output
                    need(2 * s[2], s[3], 2)
        return shapes

    def _buffers(self, B, dev):
        e = lambda *shape, dtype=BF16: torch.empty(*shape, dtype=dtype, device=dev)
        rows = B * self.hw * self.hw
        b = {"pool": {rc: [e(B, rc[0], rc[0], rc[1]) for _ in range(n)] for rc, n in self._shapes().items()},
             "img": e(B, self.H, self.W, 3), "out": e(B, self.H, self.W, 3), "recon": e(B, self.H, self.W, 3, dtype=F32),
             "mean": e(B, GROUPS, dtype=F32), "rstd": e(B, GROUPS, dtype=F32),
             "z": e(rows, self.ed, dtype=F32), "z_hi": e(rows, self.ed), "z_lo": e(rows, self.ed),
             "scores": e(rows, self.K, dtype=F32), "idx": e(rows, dtype=I32), "h_f32": e(rows, self.zc, dtype=F32)}
        widest = {}        # per attention width, its longest sequence (one width may attend at several resolutions)
        for s in self.enc + self.dec:
            if s[0] == "attn":
                widest[s[3]] = max(widest.get(s[3], 0), s[2] * s[2])
        for C, S in widest.items():
            b[("qkv", C)] = e(B * S, 3 * C)
            b[("o", C)] = e(B * S, C)
        return b

    def _alloc(self, B):
        if self._B == B:
            return
        self._B = self._b = None
        self._b = self._buffers(B, self.device)
        self._B = B

    def buffer_bytes(self, B):
        """Bytes of the buffers _alloc(B) allocates (counted on the meta device, nothing is allocated)."""
        def size(v):
            if isinstance(v, torch.Tensor):
                return v.numel() * v.element_size()
            return sum(size(x) for x in (v.values() if isinstance(v, dict) else v))
        return size(self._buffers(B, torch.device("meta")))

    def decode_pass_images(self):
        """The most images decode_tokens runs through the network at once: DECODE_PASS_BYTES of buffers."""
        return max(1, DECODE_PASS_BYTES // self.buffer_bytes(1))

    def _buf(self, res, C, *live):
        """A pooled activation [B, res, res, C] that is none of the tensors in `live`."""
        taken = {t.data_ptr() for t in live}
        for t in self._b["pool"][(res, C)]:
            if t.data_ptr() not in taken:
                return t
        raise L.DB200Error(f"VqganEngine: no free [{res}, {res}, {C}] buffer")   # _shapes under-counts: a bug

    def _desc(self, B, res, cin, cout, k, stride=1):
        key = (B, res, cin, cout, k, stride)
        d = self._descs.get(key)
        if d is None:
            d = self._descs[key] = ops.conv_desc(B, res, res, cin, cout, k, k, stride, act_f32=False)
        return d

    def _conv(self, dsc, x, name, y, residual=None):
        if y.data_ptr() == x.data_ptr():   # an implicit-GEMM conv must not overwrite the input it still reads
            raise L.DB200Error(f"VqganEngine: {name} would write its own input")
        if ops.conv_tc_supported(dsc):
            return ops.conv2d_fwd_tc(dsc, x, self.W16(name + "/weight"), self.P(name + "/bias"), residual, y)
        return ops.conv2d_fwd(dsc, x, self.P(name + "/weight"), self.P(name + "/bias"), residual, y)

    def _norm(self, x, name, y, swish):
        b = self._b
        B = x.shape[0]
        return ops.groupnorm(x, b["mean"][:B], b["rstd"][:B], self.P(name + "/weight"), self.P(name + "/bias"), y,
                             GROUPS, EPS, swish)

    # -------------------------------------------------------------------------------------------------- network
    def _resnet(self, B, name, res, cin, cout, x):
        t = self._norm(x, name + "/norm1", self._buf(res, cin, x), True)
        h = self._conv(self._desc(B, res, cin, cout, 3), t, name + "/conv1", self._buf(res, cout, x, t))
        t = self._norm(h, name + "/norm2", self._buf(res, cout, x, h), True)
        s = x
        if cin != cout:
            s = self._conv(self._desc(B, res, cin, cout, 1), x, name + "/nin_shortcut", self._buf(res, cout, h, t))
        return self._conv(self._desc(B, res, cout, cout, 3), t, name + "/conv2", self._buf(res, cout, t, s), s)

    def _attn(self, B, name, res, C, x):
        b = self._b
        rows = B * res * res
        t = self._norm(x, name + "/norm", self._buf(res, C, x), False)
        qkv, o = b[("qkv", C)][:rows], b[("o", C)][:rows]
        ops.linear_fwd(t.view(rows, C), self.qkv_w[name], qkv, bias=self.qkv_b[name])
        attn = ops.attn_noncausal if res * res <= ATTN_MAX_S else ops.attn_noncausal_long
        attn(qkv, o, B, res * res, C, C ** -0.5)
        y = self._buf(res, C, x, t)
        ops.linear_fwd(o, self.W16(name + "/proj_out/weight").view(C, C), y.view(rows, C),
                       bias=self.P(name + "/proj_out/bias"), residual=x.view(rows, C))
        return y

    def _run(self, B, steps, x):
        for s in steps:
            kind, name, res = s[:3]
            if kind == "res":
                x = self._resnet(B, name, res, s[3], s[4], x)
            elif kind == "attn":
                x = self._attn(B, name, res, s[3], x)
            elif kind == "down":   # taming pads (0, 1, 0, 1) then convolves 3x3 / 2: TF SAME at an even size
                x = self._conv(self._desc(B, res, s[3], s[3], 3, 2), x, name, self._buf(res // 2, s[3]))
            else:
                up = ops.upsample2x_fwd(x, self._buf(2 * res, s[3]))
                x = self._conv(self._desc(B, 2 * res, s[3], s[3], 3), up, name, self._buf(2 * res, s[3], up))
        return x

    def _split_mm(self, pairs, out, M, N, K, b_mn, bias=None):
        """out f32 = sum of a @ b over the listed bf16 pairs: the first product stores (+ bias), the others add into it
        in launch order, one add per element each (VaeEngine._mm_split's products)."""
        for i, (a, w) in enumerate(pairs):
            if i == 0:
                ops.gemm(a, w, out, M, N, K, a_mn=False, b_mn=b_mn, bias=bias)
            else:
                ops.gemm(a, w, out, M, N, K, a_mn=False, b_mn=b_mn, mode=L.EPI_ATOMIC, split_k=1)
        return out

    def encode_z(self, img):
        """img f32 NHWC [B, H, W, 3] in [-1, 1] -> quant_conv's output z f32 [B * h * w, embed_dim]."""
        B = img.shape[0]
        if tuple(img.shape[1:]) != (self.H, self.W, 3):
            raise L.DB200Error(f"VqganEngine: images must be [B, {self.H}, {self.W}, 3], got {tuple(img.shape)}")
        self._alloc(B)
        b = self._b
        rows = B * self.hw * self.hw
        x = ops.cast_f32_to_bf16(img.contiguous(), b["img"])
        ch = self.geo["ch"]
        x = self._conv(self._desc(B, self.H, 3, ch, 3), x, "encoder/conv_in", self._buf(self.H, ch))
        x = self._run(B, self.enc, x)
        C = self.enc_top
        t = self._norm(x, "encoder/norm_out", self._buf(self.hw, C, x), True)
        h = self._conv(self._desc(B, self.hw, C, self.zc, 3), t, "encoder/conv_out", self._buf(self.hw, self.zc, t))
        hv = h.view(rows, self.zc)     # exactly bf16: z = h @ (W_hi + W_lo) + bias
        return self._split_mm([(hv, self.qc_hi), (hv, self.qc_lo)], b["z"], rows, self.ed, self.zc, True,
                              self.P("quant_conv/bias"))

    def encode_tokens(self, img):
        """Codes of the images (first index on ties), int32 [B, image_seq_len]: the first row maximum of the scores on
        hi + lo split operands (the lo x lo product dropped).  VQ: the nearest code, score_n = z . e_n - ||e_n||^2 / 2.
        Gumbel: the mode of taming's draw, score_n = the logit z . proj_n + proj_bias_n (no noise is added)."""
        z = self.encode_z(img)
        b = self._b
        rows = z.shape[0]
        ops.split_f32(z, b["z_hi"], b["z_lo"])
        self._split_mm([(b["z_hi"], self.cb_hi), (b["z_hi"], self.cb_lo), (b["z_lo"], self.cb_hi)], b["scores"], rows,
                       self.K, self.ed, False, self.cb_bias)
        ops.argmax_rows(b["scores"], b["idx"], rows, self.K)
        return b["idx"].view(img.shape[0], self.image_seq_len)

    def decode_tokens(self, idx, offset=0):
        """Image-token ids int32 [B, image_seq_len] (minus `offset`) -> images f32 NHWC [B, H, W, 3] clamped to [-1, 1].
        Runs in passes of at most decode_pass_images() images; every launch computes an image from that image's codes
        alone, so the result does not depend on the pass size."""
        B = idx.shape[0]
        n = self.decode_pass_images()
        if B <= n:
            return self._decode_pass(idx, offset)
        out = torch.empty(B, self.H, self.W, 3, dtype=F32, device=self.device)
        for i in range(0, B, n):
            out[i:i + n].copy_(self._decode_pass(idx[i:i + n], offset))
        return out

    def _decode_pass(self, idx, offset):
        B = idx.shape[0]
        self._alloc(B)
        b = self._b
        rows = B * self.hw * self.hw
        # the codebook rows gathered exactly (as hi + lo), post_quant_conv on split operands
        ops.gather_rows_split(idx.reshape(rows).to(torch.int32).contiguous(), self.P(self.codebook), b["z_hi"],
                              b["z_lo"], offset)
        h = self._split_mm([(b["z_hi"], self.pq_hi), (b["z_hi"], self.pq_lo), (b["z_lo"], self.pq_hi)], b["h_f32"],
                           rows, self.zc, self.ed, True, self.P("post_quant_conv/bias"))
        x = ops.cast_f32_to_bf16(h, self._buf(self.hw, self.zc).view(rows, self.zc)).view(B, self.hw, self.hw, self.zc)
        C = self.enc_top
        x = self._conv(self._desc(B, self.hw, self.zc, C, 3), x, "decoder/conv_in", self._buf(self.hw, C, x))
        x = self._run(B, self.dec, x)
        C = self.dec_out_cin
        t = self._norm(x, "decoder/norm_out", self._buf(self.H, C, x), True)
        self._conv(self._desc(B, self.H, C, 3, 3), t, "decoder/conv_out", b["out"])
        return ops.clamp_bf16_to_f32(b["out"], b["recon"])
