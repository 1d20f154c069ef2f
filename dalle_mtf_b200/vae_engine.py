"""Discrete-VAE engine (host side) on the sm_90a kernels: encoder / Gumbel-softmax quantiser / decoder, forward and
backward as explicit kernel sequences, flat fp32 parameter / gradient / Adam buffers.

Mirrors src/vae_tf/models.py:46-184 (DiscreteVAE), src/vae_tf/layers.py:4-25 and the optimiser wiring of
src/model_fns_tf.py:40-66.  Parameter names are the reference's TF variable names under scope ``vae/``
(SURVEY.md Appendix B): kernels HWIO, transposed-conv kernels [kh,kw,out,in], codebook [n_hid, K].
Activations are NHWC, fp32 or bf16 (use_bf16, src/model_fns_tf.py:48-53); the codebook matmuls, Gumbel-softmax and
the loss are always fp32 (src/vae_tf/models.py:115-116,157-158).

Optional KL term (extension, kl=True; the reference has none): KL(q_r || Uniform(K)) of q_r = softmax(raw logits), the
mean over the latent rows, with a first-maximum code histogram for codebook-usage readouts (DESIGN.md §4).

Optional logit-Laplace reconstruction loss (extension, reconstruction_loss="logit_laplace"; the reference has MSE only):
the decoder's final 1x1 conv emits 2 C_p channels, mu then ln b in the packed channel order, the loss is the mean
logit-Laplace NLL of the targets mapped into (0.1, 0.9), and the image-space output is
2 clamp((sigmoid(mu) - 0.1) / 0.8, 0, 1) - 1 (DESIGN.md §4).
"""
import math

import torch

from . import lib as L
from . import ops
from .dalle_engine import ParamLayout

BF16, F32, I32 = torch.bfloat16, torch.float32, torch.int32
RECONSTRUCTION_LOSSES = ("mse", "logit_laplace")
# decode_tokens allocates every per-image buffer of the training step (_alloc), ~0.45 GiB per 256^2 image for vae_coco
# and ~1.4 GiB for the paper network, so 128 images in one pass would need 58 and 182 GiB.  Generation holds the DALL-E
# engine, its KV cache and the sampler at the same time, so decoding takes at most a fifth of an 80 GB device: passes
# of 35 and 11 images, each still thousands of pixel tiles per convolution.
DECODE_PASS_BYTES = 16 << 30


class VaeEngine:
    def __init__(self, num_tokens, image_size, convblocks, input_channels=3, use_bf16=False, recompute_grad=False,
                 stack_factor=1, device="cuda", kl=False, reconstruction_loss="mse"):
        L.require_device()
        assert math.log2(stack_factor).is_integer()                      # src/vae_tf/models.py:78
        self.K = int(num_tokens)
        # stack_factor (src/vae_tf/models.py:85-86, 155-161): the image is space_to_depth'ed on the way in and the
        # reconstruction depth_to_space'd on the way out; everything in between (and the MSE, which is a mean over the
        # same elements) works on the packed [H/s, W/s, C*s*s] tensor.  img_* = what callers see, H/W/C = packed.
        self.stack_factor = int(stack_factor)
        self.img_H = self.img_W = int(image_size)
        self.img_C = int(input_channels)
        if self.img_H % self.stack_factor != 0:
            raise L.DB200Error("image_size must be divisible by stack_factor")
        self.H = self.W = self.img_H // self.stack_factor
        self.convblocks = [(int(s), int(c)) for s, c in convblocks]
        self.C = self.img_C * self.stack_factor ** 2
        self.out_C = 2 * self.C if reconstruction_loss == "logit_laplace" else self.C   # decoder output channels
        self.use_bf16 = bool(use_bf16)
        # src/vae_tf/models.py:8-43 re-runs every residual pair inside backward to save activation memory.  Here the
        # activations are simply kept: at vae_coco (256 px, 16 images per GPU, bf16) they take ~6 GB of the 80 GB, and
        # recomputing would add a forward pass of FLOPs for nothing.  Gradients are identical either way (the
        # recomputation is deterministic), so the flag only changes memory, never numbers; model_fns says so at start-up.
        self.recompute_grad = bool(recompute_grad)
        # KL statistics buffers ([rows] lse / ent, [K] code counts) exist only when the KL term may be requested
        self.kl = bool(kl)
        self._kl_c = None
        if reconstruction_loss not in RECONSTRUCTION_LOSSES:
            raise ValueError(f"reconstruction_loss = {reconstruction_loss!r}: must be one of {RECONSTRUCTION_LOSSES}")
        self.reconstruction_loss = reconstruction_loss
        self.logit_laplace = reconstruction_loss == "logit_laplace"
        self.device = torch.device(device)
        self.act = BF16 if self.use_bf16 else F32
        if self.H % (2 ** len(self.convblocks)) != 0:
            raise L.DB200Error("image_size must be divisible by 2**len(convblocks)")
        self.n_hid = self.convblocks[-1][1]
        self.hw = self.H // (2 ** len(self.convblocks))
        self.image_seq_len = self.hw * self.hw                           # src/model_fns.py:68

        lay = ParamLayout()
        # ---- network description: list of layers with geometry
        self.enc, self.dec = [], []
        cin, res = self.C, self.H
        for b, (stack, ch) in enumerate(self.convblocks):
            for i in range(stack):
                pre = f"encoder/block_{b}/layer_{i}/"
                if i == 0:
                    lay.add(pre + "conv_downsample/kernel", (4, 4, cin, ch)); lay.add(pre + "conv_downsample/bias", (ch,))
                    self.enc.append(("down", pre + "conv_downsample", cin, ch, res))
                    res //= 2
                else:
                    for nm in ("conv_in", "conv_out"):
                        lay.add(pre + nm + "/kernel", (3, 3, ch, ch)); lay.add(pre + nm + "/bias", (ch,))
                    self.enc.append(("res", pre, ch, ch, res))
            cin = ch
        lay.add("codebook/codebook", (self.n_hid, self.K))
        for b, (stack, ch) in enumerate(reversed(self.convblocks)):
            for i in range(stack):
                pre = f"decoder/block_{b}/layer_{i}/"
                if i == 0:
                    lay.add(pre + "conv_upsample/kernel", (4, 4, ch, cin)); lay.add(pre + "conv_upsample/bias", (ch,))
                    self.dec.append(("up", pre + "conv_upsample", cin, ch, res))
                    res *= 2
                else:
                    for nm in ("conv_in", "conv_out"):
                        lay.add(pre + nm + "/kernel", (3, 3, ch, ch)); lay.add(pre + nm + "/bias", (ch,))
                    self.dec.append(("res", pre, ch, ch, res))
            cin = ch
        lay.add("decoder/conv2d/kernel", (1, 1, cin, self.out_C)); lay.add("decoder/conv2d/bias", (self.out_C,))
        self._first_dec = next(n for n in lay.order if n.startswith("decoder/"))
        self.dec_out_cin = cin
        self.layout = lay
        n = lay.size + 64
        self.n_params_padded = lay.size
        self.aux_off = lay.size
        dev = self.device
        self.master = torch.zeros(n, dtype=F32, device=dev)
        self.grads = torch.zeros(n, dtype=F32, device=dev)
        self.adam_m = torch.zeros(n, dtype=F32, device=dev)
        self.adam_v = torch.zeros(n, dtype=F32, device=dev)
        # bf16 copy of the kernels for the tensor-core convolutions (use_bf16 only)
        self.shadow = torch.zeros(n, dtype=BF16, device=dev) if self.use_bf16 else None
        # codebook matmuls: the reference keeps them in fp32 (models.py:115-118).  In bf16 mode they run on the
        # wgmma GEMM with every fp32 operand split into bf16 hi + lo parts (fp32 accumulation): ~2^-16 of sum|a||b|.
        self._cb_tc = self.use_bf16 and self.n_hid % 8 == 0 and self.K % 8 == 0
        if self._cb_tc:
            self.cb_hi = torch.zeros(self.n_hid, self.K, dtype=BF16, device=dev)
            self.cb_lo = torch.zeros(self.n_hid, self.K, dtype=BF16, device=dev)
        self._B = None
        self._grads_clean = False
        self._views = {}
        self._descs = {}

    # ------------------------------------------------------------------------------------------ parameters
    def _view(self, buf, name):
        # the per-name views are requested ~300 times per step (host time, not device time, bounds vae_example)
        key = (buf.data_ptr(), name)
        v = self._views.get(key)
        if v is None:
            v = self._views[key] = self.layout.view(buf, name)
        return v

    def P(self, name):
        return self._view(self.master, name)

    def G(self, name):
        return self._view(self.grads, name)

    def n_params(self):
        return sum(math.prod(shape) for _, shape in self.layout.entries.values())

    def W16(self, name):
        return self._view(self.shadow, name)

    def refresh_shadow(self):
        if self.shadow is not None:
            ops.cast_f32_to_bf16(self.master[:self.n_params_padded], self.shadow[:self.n_params_padded])
        if self._cb_tc:
            ops.split_f32(self.P("codebook/codebook"), self.cb_hi, self.cb_lo)

    def copy_params_from(self, src):
        """Take over the current weights of `src`, an engine of the same model (evaluation of the weights being
        trained)."""
        self.master.copy_(src.master)
        self.refresh_shadow()

    def _mm_split(self, a_parts, b_parts, out_f32, M, N, K, b_mn):
        """out = sum over the listed (a, b) pairs of a @ b on wgmma (first product stores, the rest red.add)."""
        first = True
        for a, bb in zip(a_parts, b_parts):
            if first:
                ops.gemm(a, bb, out_f32, M, N, K, a_mn=False, b_mn=b_mn)
                first = False
            else:
                ops.gemm(a, bb, out_f32, M, N, K, a_mn=False, b_mn=b_mn, mode=L.EPI_ATOMIC, split_k=1)
        return out_f32

    def _conv_fwd(self, dsc, x, name, residual, y):
        """One forward convolution: wgmma implicit GEMM when the layer qualifies (bf16, Cin % 64 == 0), else the
        shared-memory-staged direct kernel (first layer with 3 input channels, transposed convs, fp32 mode)."""
        if self.use_bf16 and ops.conv_tc_supported(dsc):
            return ops.conv2d_fwd_tc(dsc, x, self.W16(name + "/kernel"), self.P(name + "/bias"), residual, y)
        return ops.conv2d_fwd(dsc, x, self.P(name + "/kernel"), self.P(name + "/bias"), residual, y)

    def _conv_dgrad(self, dsc, dy, name, mask, dres, dx):
        if self.use_bf16 and ops.conv_dgrad_tc_supported(dsc):
            return ops.conv2d_dgrad_tc(dsc, dy, self.W16(name + "/kernel"), mask, dres, dx)
        return ops.conv2d_dgrad(dsc, dy, self.P(name + "/kernel"), mask, dres, dx)

    def _conv_wgrad(self, dsc, x, dy, name):
        if self.use_bf16 and ops.conv_wgrad_tc_supported(dsc):
            ops.conv2d_wgrad_tc(dsc, x, dy, self.G(name + "/kernel"))
            ops.colsum(dy.view(-1, dsc.Cout), self.G(name + "/bias"))       # bias gradient
        else:
            ops.conv2d_wgrad(dsc, x, dy, self.G(name + "/kernel"), self.G(name + "/bias"))

    def load_flat(self, flat, named):
        """Fill one of the flat fp32 buffers (master | adam_m | adam_v) from a dict of reference-named tensors."""
        flat.zero_()
        for name in self.layout.order:
            dst = self.layout.view(flat, name)
            t = named[name].to(device=self.device, dtype=F32)
            if tuple(t.shape) != tuple(dst.shape):
                raise L.DB200Error(f"load_params: {name}: expected {tuple(dst.shape)}, got {tuple(t.shape)}")
            dst.copy_(t)

    def load_params(self, named):
        self.load_flat(self.master, named)
        self.refresh_shadow()

    def export_params(self, source=None):
        flat = self.master if source is None else source
        return {n: self.layout.view(flat, n).detach().float().cpu().clone() for n in self.layout.order}

    def init_params(self, seed=0):
        """glorot_uniform kernels / zero biases (tf.layers defaults ‡), drawn on the device."""
        g = torch.Generator(device=self.device).manual_seed(seed)
        self.master.zero_()
        for name in self.layout.order:
            _, shape = self.layout.entries[name]
            if name.endswith("/bias"):
                continue
            if len(shape) == 4:
                rf = shape[0] * shape[1]
                fan_in, fan_out = rf * shape[2], rf * shape[3]
            else:
                fan_in, fan_out = shape
            limit = math.sqrt(6.0 / (fan_in + fan_out))
            self.P(name).copy_((torch.rand(shape, generator=g, device=self.device) * 2 - 1) * limit)
        self.refresh_shadow()

    # ------------------------------------------------------------------------------------------ buffers
    def _alloc(self, B):
        if self._B == B:
            return
        self._B = self._b = None            # the previous batch's buffers go before the new ones are allocated
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

    def _buffers(self, B, dev):
        act = self.act
        e = lambda *shape, dtype=act: torch.empty(*shape, dtype=dtype, device=dev)
        rows = B * self.hw * self.hw
        b = {"x_in": e(B, self.H, self.W, self.C), "enc": [], "dec": []}
        for kind, _, cin, ch, res in self.enc:
            if kind == "down":
                b["enc"].append({"out": e(B, res // 2, res // 2, ch)})
            else:
                b["enc"].append({"t": e(B, res, res, ch), "out": e(B, res, res, ch)})
        b.update({
            "enc_f32": e(rows, self.n_hid, dtype=F32), "logits": e(rows, self.K, dtype=F32),
            "y_soft": e(rows, self.K, dtype=F32), "y_out": e(rows, self.K, dtype=F32), "idx": e(rows, dtype=I32),
            "z_f32": e(rows, self.n_hid, dtype=F32), "z": e(B, self.hw, self.hw, self.n_hid),
        })
        for kind, _, cin, ch, res in self.dec:
            if kind == "up":
                b["dec"].append({"out": e(B, res * 2, res * 2, ch)})
            else:
                b["dec"].append({"t": e(B, res, res, ch), "out": e(B, res, res, ch)})
        if self._cb_tc:
            b.update({"y_hi": e(rows, self.K, dtype=BF16), "y_lo": e(rows, self.K, dtype=BF16),
                      "dl_hi": e(rows, self.K, dtype=BF16), "dl_lo": e(rows, self.K, dtype=BF16)})
        oc = self.out_C
        b.update({
            "recon_act": e(B, self.H, self.W, oc), "recon": e(B, self.H, self.W, oc, dtype=F32),
            "drecon": e(B, self.H, self.W, oc, dtype=F32), "drecon_act": e(B, self.H, self.W, oc),
            "dy": e(rows, self.K, dtype=F32), "dlogits": e(rows, self.K, dtype=F32),
            "dz_f32": e(rows, self.n_hid, dtype=F32), "denc_f32": e(rows, self.n_hid, dtype=F32),
        })
        if self.kl:
            b.update({"kl_lse": e(rows, dtype=F32), "kl_ent": e(rows, dtype=F32), "kl_hist": e(self.K, dtype=I32)})
        if self.logit_laplace:
            b["xhat"] = e(B, self.H, self.W, self.C, dtype=F32)      # image-space output, packed
        if self.stack_factor > 1:
            b["img_packed"] = e(B, self.H, self.W, self.C, dtype=F32)
            b["recon_flat"] = e(B, self.img_H, self.img_W, self.img_C, dtype=F32)
        # gradient scratch: two buffers per distinct activation shape
        shapes = {}
        for lst in (b["enc"], b["dec"]):
            for d in lst:
                shapes[tuple(d["out"].shape)] = None
        shapes[(B, self.hw, self.hw, self.n_hid)] = None
        b["gscratch"] = {s: [e(*s), e(*s)] for s in shapes}
        return b

    def _desc(self, B, res, cin, cout, k, stride, transposed=False, relu=False):
        key = (B, res, cin, cout, k, stride, transposed, relu)
        d = self._descs.get(key)
        if d is None:
            d = self._descs[key] = ops.conv_desc(B, res, res, cin, cout, k, k, stride, transposed=transposed,
                                                 act_f32=not self.use_bf16, relu=relu)
        return d

    def _to_act(self, src_f32, dst_act):
        if self.use_bf16:
            ops.cast_f32_to_bf16(src_f32, dst_act)
            return dst_act
        return src_f32

    def _to_f32(self, src_act, dst_f32):
        if self.use_bf16:
            ops.cast_bf16_to_f32(src_act, dst_f32)
            return dst_f32
        return src_act

    # ------------------------------------------------------------------------------------------ forward
    def _res_fwd(self, B, pre, ch, res, x, sv):
        """x + conv_out(relu(conv_in(x)))   (src/vae_tf/models.py:99-109 / 143-153)."""
        self._conv_fwd(self._desc(B, res, ch, ch, 3, 1, relu=True), x, pre + "conv_in", None, sv["t"])
        self._conv_fwd(self._desc(B, res, ch, ch, 3, 1), sv["t"], pre + "conv_out", x, sv["out"])
        return sv["out"]

    def encode_logits(self, img, for_training=False):
        """DiscreteVAE.encoder (src/vae_tf/models.py:81-120): img fp32 NHWC [B,H,W,C] -> fp32 logits [B*h*w, K]."""
        B = img.shape[0]
        self._alloc(B)
        b = self._b
        img = self._pack(img)
        # bf16 inference path: the first layer reads the fp32 image directly (dedicated kernel, cast fused)
        first_direct = (self.use_bf16 and not for_training and self.C == 3 and self.enc[0][0] == "down" and
                        self.enc[0][3] % 64 == 0 and self.H % 2 == 0)
        x = img if first_direct else self._to_act(img, b["x_in"])
        self._x0 = x
        for li, ((kind, name, cin, ch, res), sv) in enumerate(zip(self.enc, b["enc"])):
            if li == 0 and first_direct:
                ops.conv2d_first_fwd(img, self.P(name + "/kernel"), self.P(name + "/bias"), sv["out"])
                x = sv["out"]
            elif kind == "down":
                self._conv_fwd(self._desc(B, res, cin, ch, 4, 2), x, name, None, sv["out"])
                x = sv["out"]
            else:
                x = self._res_fwd(B, name, ch, res, x, sv)
        return self._codebook_logits(x, B * self.hw * self.hw)

    def _codebook_logits(self, x, rows):
        """logits = enc @ codebook (src/vae_tf/models.py:115-118) for the encoder output x (activation dtype)."""
        b = self._b
        if self._cb_tc:   # x is exactly bf16: logits = x @ (C_hi + C_lo)
            xb = x.view(rows, self.n_hid)
            self._enc_bf16 = xb
            self._mm_split([xb, xb], [self.cb_hi, self.cb_lo], b["logits"], rows, self.K, self.n_hid, b_mn=True)
            return b["logits"]
        xf = self._to_f32(x.view(rows, self.n_hid), b["enc_f32"])
        self._enc_f32 = xf
        ops.rowmatmul(xf, self.P("codebook/codebook"), b["logits"], rows, self.n_hid, self.K)
        return b["logits"]

    def encode_tokens(self, img):
        """src/model_fns.py:72-77: argmax over the K codes (first maximum), int32 [B, image_seq_len]."""
        logits = self.encode_logits(img)
        rows = logits.shape[0]
        ops.argmax_rows(logits, self._b["idx"], rows, self.K)
        return self._b["idx"].view(img.shape[0], self.image_seq_len)

    def _decode_from_z(self, B):
        """DiscreteVAE.decoder after the tied codebook matmul (src/vae_tf/models.py:129-163): b["z_f32"] -> recon fp32
        (logit-Laplace: the packed stats, mu | ln b)."""
        b = self._b
        rows = B * self.hw * self.hw
        x = self._to_act(b["z_f32"], b["z"].view(rows, self.n_hid)).view(B, self.hw, self.hw, self.n_hid)
        self._z = x
        for (kind, name, cin, ch, res), sv in zip(self.dec, b["dec"]):
            if kind == "up":
                self._conv_fwd(self._desc(B, res, cin, ch, 4, 2, transposed=True), x, name, None, sv["out"])
                x = sv["out"]
            else:
                x = self._res_fwd(B, name, ch, res, x, sv)
        self._dec_last = x
        ops.conv2d_fwd(self._desc(B, self.H, self.dec_out_cin, self.out_C, 1, 1), x, self.P("decoder/conv2d/kernel"),
                       self.P("decoder/conv2d/bias"), None, b["recon_act"])                   # models.py:155
        return self._to_f32(b["recon_act"], b["recon"])

    def _pack(self, img):
        """space_to_depth of the caller's image (no-op for stack_factor 1)."""
        if self.stack_factor == 1:
            return img
        return ops.space_to_depth(img.view(-1, self.img_H, self.img_W, self.img_C), self._b["img_packed"],
                                  self.stack_factor)

    def _unpack(self, recon):
        """depth_to_space of the packed reconstruction for the caller (no-op for stack_factor 1)."""
        if self.stack_factor == 1:
            return recon
        return ops.space_to_depth(recon, self._b["recon_flat"], self.stack_factor, inverse=True)

    def _codebook_lookup(self, B):
        """z = y @ codebook^T for b["y_out"] (src/vae_tf/models.py:127, tied weight)."""
        b = self._b
        rows = B * self.hw * self.hw
        if self._cb_tc:
            # z = y @ C^T with y, C split into bf16 hi + lo.  |lo| <= 2^-8 |x| and x - hi - lo <= 2^-16 |x|, so the
            # dropped lo*lo term and the two split residuals cost <= 3.1 * 2^-16 * sum|y||C| per element: ~2^-16
            # relative, not fp32's 2^-24 (tests/test_vae_kernels_gpu.py holds the products to that bound)
            ops.split_f32(b["y_out"], b["y_hi"], b["y_lo"])
            self._mm_split([b["y_hi"], b["y_hi"], b["y_lo"]], [self.cb_hi, self.cb_lo, self.cb_hi], b["z_f32"], rows,
                           self.n_hid, self.K, b_mn=False)
        else:
            ops.rowmatmul(b["y_out"], self.P("codebook/codebook"), b["z_f32"], rows, self.K, self.n_hid,
                          b_transposed=True)

    def decode_tokens(self, idx, offset=0):
        """Image-token ids int32 [B, image_seq_len] (minus `offset`) -> reconstruction fp32 NHWC [B,H,W,C] in [-1,1]-ish:
        one-hot codes through the tied codebook and the decoder — the generation-side counterpart of encode_tokens.

        Runs in passes of at most decode_pass_images() images, each written into one output tensor; every decode launch
        computes an image from that image's codes alone, so the result does not depend on the pass size."""
        B = idx.shape[0]
        n = self.decode_pass_images()
        if B <= n:
            return self._decode_pass(idx, offset)
        out = torch.empty(B, self.img_H, self.img_W, self.img_C, dtype=F32, device=self.device)
        for i in range(0, B, n):
            out[i:i + n].copy_(self._decode_pass(idx[i:i + n], offset))
        return out

    def _decode_pass(self, idx, offset):
        B = idx.shape[0]
        self._alloc(B)
        rows = B * self.hw * self.hw
        ops.onehot_rows(idx.reshape(rows).contiguous(), self._b["y_out"], offset)
        self._codebook_lookup(B)
        out = self._decode_from_z(B)
        if self.logit_laplace:
            n_pix = B * self.H * self.W
            ops.logit_laplace(out, None, None, self._b["xhat"], None, None, n_pix, self.C, 0.0)
            out = self._b["xhat"]
        return self._unpack(out)

    def forward(self, img, u, temperature=1.0, hard=True, loss_accum=None, kl_weight=None, kl_accum=None,
                mse_accum=None):
        """DiscreteVAE.forward(return_recon_loss=True) (src/vae_tf/models.py:165-184).  u: fp32 uniform noise
        [B*h*w, K] in [1e-9, 1) or None (no noise).  Adds sum((img-out)^2)/numel into loss_accum; returns recon.

        Logit-Laplace engine: adds the mean NLL into loss_accum (default aux slot 0) and the mean (xhat - img)^2 into
        mse_accum (default aux slot 2), and returns the image-space output xhat.

        kl_weight (engine built with kl=True; None = no KL statistics): also adds the mean over the B*h*w latent rows of
        KL(softmax(logits) || Uniform(K)) into kl_accum (default: aux slot 1, behind the loss), counts the first-maximum
        code of every row into code_counts(), and, when kl_weight > 0, makes backward add the gradient of
        kl_weight * KL to the encoder logits'."""
        B = img.shape[0]
        logits = self.encode_logits(img, for_training=True)
        b = self._b
        rows = B * self.hw * self.hw
        self._tau = float(temperature)
        self._kl_c = None
        if kl_weight is not None:
            if not self.kl:
                raise L.DB200Error("VaeEngine.forward: kl_weight needs an engine built with kl=True")
            if kl_accum is None:
                kl_accum = self.grads[self.aux_off + 1:self.aux_off + 2]
            b["kl_hist"].zero_()
            ops.vae_kl_stats(logits, b["kl_lse"], b["kl_ent"], b["kl_hist"], kl_accum, rows, self.K, 1.0 / rows)
            if kl_weight > 0:   # weight 0 monitors only: backward then runs exactly the plain kernels
                self._kl_c = float(kl_weight) / rows
        ops.gumbel_softmax_fwd(logits, u, b["y_soft"], b["y_out"], b["idx"], rows, self.K, self._tau, hard)
        self._codebook_lookup(B)
        recon = self._decode_from_z(B)
        self._img = img
        if loss_accum is None:
            loss_accum = self.grads[self.aux_off:self.aux_off + 1]
        n = img.numel()
        self._loss_scale = 1.0 / n
        packed = self._b["img_packed"] if self.stack_factor > 1 else img   # written by encode_logits
        if self.logit_laplace:
            if mse_accum is None:
                mse_accum = self.grads[self.aux_off + 2:self.aux_off + 3]
            ops.logit_laplace(recon, packed, b["drecon"], b["xhat"], loss_accum, mse_accum, B * self.H * self.W,
                              self.C, 1.0 / n)
            return self._unpack(b["xhat"])
        ops.mse_fwd_bwd(recon, packed, b["drecon"], loss_accum, 1.0 / n)                       # layers.py:24-25
        return self._unpack(recon)

    # ------------------------------------------------------------------------------------------ backward
    def _res_bwd(self, B, pre, ch, res, x_in, sv, dx, scratch):
        """Backward of x_out = x_in + conv_out(t), t = relu(conv_in(x_in)); dx is overwritten with d(x_in)."""
        d_out = self._desc(B, res, ch, ch, 3, 1)
        self._conv_wgrad(d_out, sv["t"], dx, pre + "conv_out")
        dt = scratch
        self._conv_dgrad(d_out, dx, pre + "conv_out", sv["t"], None, dt)                     # masked by t > 0
        self._conv_wgrad(d_out, x_in, dt, pre + "conv_in")
        # d(x_in) = dgrad(conv_in)(dt) + dx: read dx as the residual and write the result in place
        self._conv_dgrad(d_out, dt, pre + "conv_in", None, dx, dx)
        return dx

    def backward(self, grad_scale=1.0, on_bucket_ready=None):
        """Back-propagates d(loss) * grad_scale; gradients ACCUMULATE into self.grads.
        on_bucket_ready(start, end) is called as soon as the flat range [start, end) is final (data-parallel hook):
        decoder (+ the aux loss slot) first, then the codebook, then the encoder — the flat buffer is in forward
        order, so backward completes it from the tail and each range is reduced while the rest still runs."""
        b = self._b
        B = self._img.shape[0]
        rows = B * self.hw * self.hw
        if grad_scale != 1.0:
            raise L.DB200Error("VaeEngine.backward: fold grad_scale into the Adam step (grad_scale argument there)")
        dx = self._to_act(b["drecon"], b["drecon_act"])
        d1 = self._desc(B, self.H, self.dec_out_cin, self.out_C, 1, 1)
        ops.conv2d_wgrad(d1, self._dec_last, dx, self.G("decoder/conv2d/kernel"), self.G("decoder/conv2d/bias"))
        gs = b["gscratch"][tuple(self._dec_last.shape)]
        ops.conv2d_dgrad(d1, dx, self.P("decoder/conv2d/kernel"), None, None, gs[0])
        dx = gs[0]
        # decoder, reversed
        inputs = [self._z] + [sv["out"] for sv in b["dec"][:-1]]
        for (kind, name, cin, ch, res), sv, x_in in reversed(list(zip(self.dec, b["dec"], inputs))):
            if kind == "up":
                dsc = self._desc(B, res, cin, ch, 4, 2, transposed=True)
                self._conv_wgrad(dsc, x_in, dx, name)
                nxt = b["gscratch"][tuple(x_in.shape)][0]
                self._conv_dgrad(dsc, dx, name, None, None, nxt)
                dx = nxt
            else:
                pair = b["gscratch"][tuple(x_in.shape)]
                scratch = pair[1] if dx is pair[0] else pair[0]
                dx = self._res_bwd(B, name, ch, res, x_in, sv, dx, scratch)
        if on_bucket_ready:
            s0, _ = self.layout.span(self._first_dec, self._first_dec)
            _, e0 = self.layout.span("decoder/conv2d/bias", "decoder/conv2d/bias")
            on_bucket_ready(s0, e0 + 64)      # + the aux scalars (loss) behind the last parameter
        self._quantiser_backward(dx, rows)
        if on_bucket_ready:
            on_bucket_ready(*self.layout.span("codebook/codebook", "codebook/codebook"))
        pair = b["gscratch"][(B, self.hw, self.hw, self.n_hid)]
        dx = self._to_act(b["denc_f32"], pair[0].view(rows, self.n_hid)).view(B, self.hw, self.hw, self.n_hid)
        if not self.use_bf16:
            dx = b["denc_f32"].view(B, self.hw, self.hw, self.n_hid)
        # encoder, reversed
        inputs = [self._x0] + [sv["out"] for sv in b["enc"][:-1]]
        for li, ((kind, name, cin, ch, res), sv, x_in) in reversed(list(enumerate(zip(self.enc, b["enc"], inputs)))):
            if kind == "down":
                dsc = self._desc(B, res, cin, ch, 4, 2)
                self._conv_wgrad(dsc, x_in, dx, name)
                if li > 0:  # the gradient w.r.t. the image itself is never needed
                    nxt = b["gscratch"][tuple(x_in.shape)][0]
                    self._conv_dgrad(dsc, dx, name, None, None, nxt)
                    dx = nxt
            else:
                pair = b["gscratch"][tuple(x_in.shape)]
                if dx is not pair[0] and dx is not pair[1]:  # fp32 path: dx is denc_f32 viewed; move into a pair slot
                    pair[0].copy_(dx)
                    dx = pair[0]
                scratch = pair[1] if dx is pair[0] else pair[0]
                dx = self._res_bwd(B, name, ch, res, x_in, sv, dx, scratch)
        if on_bucket_ready:
            s0, _ = self.layout.span(self.layout.order[0], self.layout.order[0])
            e0, _ = self.layout.span("codebook/codebook", "codebook/codebook")
            on_bucket_ready(s0, e0)

    def _quantiser_backward(self, dx, rows):
        """Backward of z = y_out @ codebook^T and of the straight-through Gumbel softmax, for dx = d(loss)/dz: adds the
        codebook gradient (decode and encode side) into self.grads and leaves d(encoder output) in b["denc_f32"]."""
        b = self._b
        cb = self.P("codebook/codebook")
        gcb = self.G("codebook/codebook")
        if self._cb_tc:
            dzb = dx.view(rows, self.n_hid)                                                       # exactly bf16
            ops.linear_wgrad(dzb, b["y_hi"], gcb); ops.linear_wgrad(dzb, b["y_lo"], gcb)          # d codebook (decode)
            self._mm_split([dzb, dzb], [self.cb_hi, self.cb_lo], b["dy"], rows, self.K, self.n_hid, b_mn=True)
            self._gumbel_backward(rows)
            ops.split_f32(b["dlogits"], b["dl_hi"], b["dl_lo"])
            ops.linear_wgrad(self._enc_bf16, b["dl_hi"], gcb); ops.linear_wgrad(self._enc_bf16, b["dl_lo"], gcb)
            self._mm_split([b["dl_hi"], b["dl_hi"], b["dl_lo"]], [self.cb_hi, self.cb_lo, self.cb_hi],
                           b["denc_f32"], rows, self.n_hid, self.K, b_mn=False)
        else:
            dz = self._to_f32(dx.view(rows, self.n_hid), b["dz_f32"])
            ops.rowmatmul_tn(dz, b["y_out"], gcb, rows, self.n_hid, self.K)                       # d codebook (decode)
            ops.rowmatmul(dz, cb, b["dy"], rows, self.n_hid, self.K)                              # dy = dz @ C
            self._gumbel_backward(rows)
            ops.rowmatmul_tn(self._enc_f32, b["dlogits"], gcb, rows, self.n_hid, self.K)
            ops.rowmatmul(b["dlogits"], cb, b["denc_f32"], rows, self.K, self.n_hid, b_transposed=True)

    def _gumbel_backward(self, rows):
        """b["dlogits"] from b["dy"]: the straight-through Gumbel-softmax backward, plus the gradient of
        kl_weight * KL (kl_weight / rows * q (l - lse - ent)) in the same pass when forward was given kl_weight > 0."""
        b = self._b
        if self._kl_c is None:
            ops.gumbel_softmax_bwd(b["y_soft"], b["dy"], b["dlogits"], rows, self.K, self._tau)   # straight-through
        else:
            ops.gumbel_softmax_bwd_kl(b["y_soft"], b["dy"], b["logits"], b["kl_lse"], b["kl_ent"], b["dlogits"], rows,
                                      self.K, self._tau, self._kl_c)

    def code_counts(self):
        """int32 [K]: how many latent rows of the last forward with kl_weight had each code as the first maximum of
        their logits (a row with a NaN counts as code 0)."""
        return self._b["kl_hist"]

    # ------------------------------------------------------------------------------------------ optimiser
    def zero_grads(self):
        """See DalleEngine.zero_grads: the Adam kernel leaves the gradient buffer zeroed behind itself."""
        if self._grads_clean:
            self.grads[self.aux_off:].zero_()
        else:
            self.grads.zero_()
        self._grads_clean = False

    def optimizer_step(self, lr, step, grad_scale=1.0, beta1=0.9, beta2=0.999, eps=1e-8):
        """tf.train.AdamOptimizer (bias-corrected, no clipping), src/model_fns_tf.py:58-66.  `step` = t >= 1.
        grad_scale = 1/world_size turns the all-reduced SUM into CrossShardOptimizer's mean."""
        n = self.n_params_padded
        ops.adam_step(self.master[:n], self.adam_m[:n], self.adam_v[:n], self.grads[:n],
                      None if self.shadow is None else self.shadow[:n], lr, beta1, beta2, eps, 0.0, None, 0.0,
                      grad_scale, True, step, zero_grad=True)
        self._grads_clean = True
        if self._cb_tc:
            ops.split_f32(self.P("codebook/codebook"), self.cb_hi, self.cb_lo)


def codebook_usage(counts):
    """(codes_used, perplexity) of a code histogram: the number of codes with a count > 0 and exp(-sum p log p),
    p = counts / sum(counts).  Host values (reading a device histogram synchronises)."""
    c = counts.detach().double().cpu()
    n = c.sum()
    p = c[c > 0] / n
    return int((c > 0).sum()), float(torch.exp(-(p * p.log()).sum()))
