"""Discrete-VAE engine of the DALL-E paper's network (architecture "dalle_paper"; the reference's network is
vae_engine.VaeEngine's).  DESIGN.md §4 and oracle/vae_paper.py hold the definition:

  block y = id(x) + gain * res(x), gain = 1 / (group_count * n_blk_per_group)^2, res = four convs, each reading the
  ReLU of what precedes it (pre-activation); encoder: 7x7 input conv, groups of blocks with 2x2 max-pools between them,
  ReLU + an f32 1x1 projection to the logits; decoder: an f32 1x1 projection of the quantiser's one-hot (its own weights,
  not tied to the encoder), groups of blocks with 2x nearest upsampling between them, ReLU + a 1x1 conv to C (MSE) or
  2 C (logit-Laplace) channels.

The quantiser, the losses, the KL statistics, the flat buffers and the optimiser are VaeEngine's: this class replaces
the network on either side of the [rows, num_tokens] logits and nothing else.  Every step runs on the library's
kernels: the block convs on K11 (wgmma when the shape qualifies), the 7x7 conv, pool, upsample and the residual / ReLU
pointwise step on K11p, the two projections on the bf16 hi + lo split GEMM in bf16 mode (on the f32 conv kernels in f32
mode).
"""
import math

import torch

from . import lib as L
from . import ops
from .dalle_engine import ParamLayout
from .vae_engine import BF16, F32, I32, RECONSTRUCTION_LOSSES, VaeEngine


def check_paper_geometry(image_size, n_hid, n_blk_per_group, group_count, n_init):
    """Raises ValueError for a geometry the paper's network does not define."""
    for k, v in (("image_size", image_size), ("n_hid", n_hid), ("n_blk_per_group", n_blk_per_group),
                 ("group_count", group_count), ("n_init", n_init)):
        if isinstance(v, bool) or not isinstance(v, int) or v < 1:
            raise ValueError(f"{k} = {v!r}: must be an integer >= 1")
    if n_hid % 8 or n_hid < 64:
        raise ValueError(f"n_hid = {n_hid}: must be a multiple of 8 and >= 64 (the bottleneck width is width / 4)")
    if n_init % 8:
        raise ValueError(f"n_init = {n_init}: must be a multiple of 8")
    if image_size % (2 ** (group_count - 1)):
        raise ValueError(f"image_size = {image_size} is not divisible by 2^(group_count - 1) = "
                         f"{2 ** (group_count - 1)}")


class PaperVaeEngine(VaeEngine):
    def __init__(self, num_tokens, image_size, input_channels=3, n_hid=256, n_blk_per_group=2, group_count=4,
                 n_init=128, use_bf16=False, recompute_grad=False, device="cuda", kl=False, reconstruction_loss="mse"):
        L.require_device()
        check_paper_geometry(image_size, n_hid, n_blk_per_group, group_count, n_init)
        if reconstruction_loss not in RECONSTRUCTION_LOSSES:
            raise ValueError(f"reconstruction_loss = {reconstruction_loss!r}: must be one of {RECONSTRUCTION_LOSSES}")
        self.K = int(num_tokens)
        self.stack_factor = 1
        self.img_H = self.img_W = self.H = self.W = int(image_size)
        self.img_C = self.C = int(input_channels)
        if not 1 <= self.C <= 4:
            raise L.DB200Error(f"input_channels = {self.C}: the 7x7 input conv covers 1 to 4 channels")
        self.reconstruction_loss = reconstruction_loss
        self.logit_laplace = reconstruction_loss == "logit_laplace"
        self.out_C = 2 * self.C if self.logit_laplace else self.C
        self.use_bf16 = bool(use_bf16)
        if self.use_bf16 and self.K % 8:
            raise L.DB200Error(f"num_tokens = {self.K}: the bf16 projections need a multiple of 8")
        self.recompute_grad = bool(recompute_grad)   # as VaeEngine: activations are kept, the flag changes nothing
        self.kl = bool(kl)
        self._kl_c = None
        self.device = torch.device(device)
        self.act = BF16 if self.use_bf16 else F32
        self.convblocks = None
        self.base_width, self.n_blk_per_group, self.group_count, self.n_init = n_hid, n_blk_per_group, group_count, \
            n_init
        self.gain = 1.0 / (group_count * n_blk_per_group) ** 2
        self.hw = self.H // 2 ** (group_count - 1)
        self.image_seq_len = self.hw * self.hw
        self.n_hid = 2 ** (group_count - 1) * n_hid          # encoder output width (what the projection reads)
        self.dec_out_cin = n_hid

        lay = ParamLayout()

        def conv(name, k, cin, cout):
            lay.add(name + "/kernel", (k, k, cin, cout)); lay.add(name + "/bias", (cout,))

        # blocks: (prefix, n_in, n_out, kernel sizes, resolution, resample after it: "pool" | "up" | None)
        self.enc, self.dec = [], []
        conv("encoder/input", 7, self.C, n_hid)
        for side in ("encoder", "decoder"):
            if side == "encoder":
                prev, res, ks, blocks = n_hid, self.H, (3, 3, 3, 1), self.enc
                widths = [2 ** (k - 1) * n_hid for k in range(1, group_count + 1)]
            else:
                conv("decoder/input", 1, self.K, n_init)
                prev, res, ks, blocks = n_init, self.hw, (1, 3, 3, 3), self.dec
                widths = [2 ** (group_count - k) * n_hid for k in range(1, group_count + 1)]
            for k, w in enumerate(widths, 1):
                for i in range(1, n_blk_per_group + 1):
                    pre = f"{side}/group_{k}/block_{i}/"
                    n_in = prev if i == 1 else w
                    if n_in != w:
                        conv(pre + "id_path", 1, n_in, w)
                    chans = (n_in, w // 4, w // 4, w // 4, w)
                    for j in range(4):
                        conv(pre + f"res_path/conv_{j + 1}", ks[j], chans[j], chans[j + 1])
                    last = i == n_blk_per_group and k < group_count
                    blocks.append((pre, n_in, w, ks, res, ("pool" if side == "encoder" else "up") if last else None))
                prev = w
                if k < group_count:
                    res = res // 2 if side == "encoder" else res * 2
            if side == "encoder":
                conv("encoder/output/conv", 1, self.n_hid, self.K)
        conv("decoder/output/conv", 1, n_hid, self.out_C)
        self.layout = lay
        n = lay.size + 64
        self.n_params_padded = lay.size
        self.aux_off = lay.size
        dev = self.device
        self.master = torch.zeros(n, dtype=F32, device=dev)
        self.grads = torch.zeros(n, dtype=F32, device=dev)
        self.adam_m = torch.zeros(n, dtype=F32, device=dev)
        self.adam_v = torch.zeros(n, dtype=F32, device=dev)
        self.shadow = torch.zeros(n, dtype=BF16, device=dev) if self.use_bf16 else None
        self._cb_tc = False   # no codebook: the projections below take its place
        if self.use_bf16:     # f32 projections as bf16 hi + lo operands of the wgmma GEMM (VaeEngine's codebook split)
            self.eo_hi = torch.zeros(self.n_hid, self.K, dtype=BF16, device=dev)
            self.eo_lo = torch.zeros(self.n_hid, self.K, dtype=BF16, device=dev)
            self.di_hi = torch.zeros(self.K, n_init, dtype=BF16, device=dev)
            self.di_lo = torch.zeros(self.K, n_init, dtype=BF16, device=dev)
        self._B = None
        self._grads_clean = False
        self._views = {}
        self._descs = {}
        self._pool = {}

    # ------------------------------------------------------------------------------------------ parameters
    def refresh_shadow(self):
        if self.shadow is not None:
            ops.cast_f32_to_bf16(self.master[:self.n_params_padded], self.shadow[:self.n_params_padded])
            self._split_projections()

    def _split_projections(self):
        ops.split_f32(self.P("encoder/output/conv/kernel"), self.eo_hi, self.eo_lo)
        ops.split_f32(self.P("decoder/input/kernel"), self.di_hi, self.di_lo)

    def init_params(self, seed=0):
        """Normal kernels with std 1 / sqrt(cin kh kw), zero biases, drawn on the device."""
        g = torch.Generator(device=self.device).manual_seed(seed)
        self.master.zero_()
        for name in self.layout.order:
            _, shape = self.layout.entries[name]
            if name.endswith("/kernel"):
                std = 1.0 / math.sqrt(shape[0] * shape[1] * shape[2])
                self.P(name).copy_(torch.randn(shape, generator=g, device=self.device) * std)
        self.refresh_shadow()

    def optimizer_step(self, lr, step, grad_scale=1.0, beta1=0.9, beta2=0.999, eps=1e-8):
        super().optimizer_step(lr, step, grad_scale, beta1, beta2, eps)
        if self.use_bf16:
            self._split_projections()

    # ------------------------------------------------------------------------------------------ buffers
    def _alloc(self, B):
        if self._B == B:
            return
        dev, act = self.device, self.act
        e = lambda *shape, dtype=act: torch.empty(*shape, dtype=dtype, device=dev)
        self._B = B
        rows = B * self.hw * self.hw
        b = {"x0": e(B, self.H, self.W, self.base_width), "enc": [], "dec": []}
        for side in ("enc", "dec"):
            for pre, n_in, n_out, ks, res, after in getattr(self, side):
                sv = {"a": e(B, res, res, n_in), "r": e(B, res, res, n_out), "y": e(B, res, res, n_out)}
                for j in (1, 2, 3):
                    sv[f"t{j}"] = e(B, res, res, n_out // 4)
                if n_in != n_out:
                    sv["id"] = e(B, res, res, n_out)
                if after == "pool":
                    sv["pool"] = e(B, res // 2, res // 2, n_out)
                elif after == "up":
                    sv["up"] = e(B, res * 2, res * 2, n_out)
                b[side].append(sv)
        K = self.K
        b.update({
            "enc_relu": e(B, self.hw, self.hw, self.n_hid), "logits": e(rows, K, dtype=F32),
            "y_soft": e(rows, K, dtype=F32), "y_out": e(rows, K, dtype=F32), "idx": e(rows, dtype=I32),
            "z_f32": e(rows, self.n_init, dtype=F32), "z": e(B, self.hw, self.hw, self.n_init),
            "dec_relu": e(B, self.H, self.W, self.dec_out_cin),
            "recon_act": e(B, self.H, self.W, self.out_C), "recon": e(B, self.H, self.W, self.out_C, dtype=F32),
            "drecon": e(B, self.H, self.W, self.out_C, dtype=F32), "drecon_act": e(B, self.H, self.W, self.out_C),
            "dy": e(rows, K, dtype=F32), "dlogits": e(rows, K, dtype=F32), "denc_f32": e(rows, self.n_hid, dtype=F32),
        })
        if self.use_bf16:
            b.update({"y_hi": e(rows, K, dtype=BF16), "y_lo": e(rows, K, dtype=BF16),
                      "dl_hi": e(rows, K, dtype=BF16), "dl_lo": e(rows, K, dtype=BF16)})
        if self.kl:
            b.update({"kl_lse": e(rows, dtype=F32), "kl_ent": e(rows, dtype=F32), "kl_hist": e(K, dtype=I32)})
        if self.logit_laplace:
            b["xhat"] = e(B, self.H, self.W, self.C, dtype=F32)
        self._b = b
        self._pool = {}

    def _scratch(self, shape, avoid=()):
        """A gradient buffer of `shape` (activation dtype) other than the tensors in `avoid`; the pool grows to the
        number of buffers of one shape that are alive at once (at most three) and is reused from step to step."""
        shape = tuple(shape)
        taken = {t.data_ptr() for t in avoid}
        lst = self._pool.setdefault(shape, [])
        for t in lst:
            if t.data_ptr() not in taken:
                return t
        t = torch.empty(shape, dtype=self.act, device=self.device)
        lst.append(t)
        return t

    # ------------------------------------------------------------------------------------------ forward
    def _block_fwd(self, B, blk, x, sv):
        """y = id(x) + gain * (conv_4(relu(conv_3(relu(conv_2(relu(conv_1(relu(x)))))))) + b_4)."""
        pre, n_in, n_out, ks, res, _ = blk
        h = n_out // 4
        ops.residual_gain(x, 1.0, relu_y=sv["a"])
        t, chans = sv["a"], (n_in, h, h, h)
        for j in range(3):
            self._conv_fwd(self._desc(B, res, chans[j], h, ks[j], 1, relu=True), t, pre + f"res_path/conv_{j + 1}",
                           None, sv[f"t{j + 1}"])
            t = sv[f"t{j + 1}"]
        self._conv_fwd(self._desc(B, res, h, n_out, ks[3], 1), t, pre + "res_path/conv_4", None, sv["r"])
        idv = x
        if n_in != n_out:
            self._conv_fwd(self._desc(B, res, n_in, n_out, 1, 1), x, pre + "id_path", None, sv["id"])
            idv = sv["id"]
        return ops.residual_gain(sv["r"], self.gain, id=idv, y=sv["y"])

    def encode_logits(self, img, for_training=False):
        """img f32 NHWC [B,H,W,C] in [-1, 1] -> f32 logits [B*h*w, K]."""
        B = img.shape[0]
        self._alloc(B)
        b = self._b
        self._img_in = img
        x = ops.conv7x7_in_fwd(img, self.P("encoder/input/kernel"), self.P("encoder/input/bias"), b["x0"])
        for blk, sv in zip(self.enc, b["enc"]):
            x = self._block_fwd(B, blk, x, sv)
            if blk[5] == "pool":
                x = ops.maxpool2x2_fwd(x, sv["pool"])
        self._enc_last = x
        ops.residual_gain(x, 1.0, relu_y=b["enc_relu"])
        rows = B * self.hw * self.hw
        bias = self.P("encoder/output/conv/bias")
        if self.use_bf16:   # relu(x) is exactly bf16: logits = a @ (W_hi + W_lo) + bias
            a = b["enc_relu"].view(rows, self.n_hid)
            ops.gemm(a, self.eo_hi, b["logits"], rows, self.K, self.n_hid, a_mn=False, b_mn=True, bias=bias)
            ops.gemm(a, self.eo_lo, b["logits"], rows, self.K, self.n_hid, a_mn=False, b_mn=True, mode=L.EPI_ATOMIC,
                     split_k=1)
        else:
            ops.conv2d_fwd(self._desc(B, self.hw, self.n_hid, self.K, 1, 1), b["enc_relu"],
                           self.P("encoder/output/conv/kernel"), bias, None, b["logits"])
        return b["logits"]

    def _codebook_lookup(self, B):
        """The decoder's input projection: b["z_f32"] = b["y_out"] @ W_in + b_in (f32)."""
        b = self._b
        rows = B * self.hw * self.hw
        bias = self.P("decoder/input/bias")
        if self.use_bf16:   # y and W split into bf16 hi + lo; the lo * lo product is dropped (VaeEngine's codebook)
            ops.split_f32(b["y_out"], b["y_hi"], b["y_lo"])
            for i, (a, w) in enumerate(((b["y_hi"], self.di_hi), (b["y_hi"], self.di_lo), (b["y_lo"], self.di_hi))):
                if i == 0:
                    ops.gemm(a, w, b["z_f32"], rows, self.n_init, self.K, a_mn=False, b_mn=True, bias=bias)
                else:
                    ops.gemm(a, w, b["z_f32"], rows, self.n_init, self.K, a_mn=False, b_mn=True, mode=L.EPI_ATOMIC,
                             split_k=1)
        else:
            ops.conv2d_fwd(self._desc(B, self.hw, self.K, self.n_init, 1, 1), b["y_out"],
                           self.P("decoder/input/kernel"), bias, None, b["z_f32"])

    def _decode_from_z(self, B):
        """b["z_f32"] -> the decoder output f32 [B,H,W,out_C]."""
        b = self._b
        rows = B * self.hw * self.hw
        x = self._to_act(b["z_f32"], b["z"].view(rows, self.n_init)).view(B, self.hw, self.hw, self.n_init)
        self._z = x
        for blk, sv in zip(self.dec, b["dec"]):
            x = self._block_fwd(B, blk, x, sv)
            if blk[5] == "up":
                x = ops.upsample2x_fwd(x, sv["up"])
        self._dec_last = x
        ops.residual_gain(x, 1.0, relu_y=b["dec_relu"])
        ops.conv2d_fwd(self._desc(B, self.H, self.dec_out_cin, self.out_C, 1, 1), b["dec_relu"],
                       self.P("decoder/output/conv/kernel"), self.P("decoder/output/conv/bias"), None, b["recon_act"])
        return self._to_f32(b["recon_act"], b["recon"])

    # ------------------------------------------------------------------------------------------ backward
    def _block_bwd(self, B, blk, x, sv, dy):
        """Gradients of one block's parameters from dy = d(loss)/d(y) (a scratch buffer, consumed); returns
        d(loss)/d(x) = (x > 0) dgrad(conv_1) + d(id)."""
        pre, n_in, n_out, ks, res, _ = blk
        h = n_out // 4
        g = ops.residual_gain(dy, self.gain, y=self._scratch(dy.shape, (dy,)))        # d(conv_4 + b_4)
        ins, chans = (sv["a"], sv["t1"], sv["t2"], sv["t3"]), (n_in, h, h, h, n_out)
        for j in (3, 2, 1):
            dsc, name = self._desc(B, res, chans[j], chans[j + 1], ks[j], 1), pre + f"res_path/conv_{j + 1}"
            self._conv_wgrad(dsc, ins[j], g, name)
            nxt = self._scratch(ins[j].shape, (g, dy))
            self._conv_dgrad(dsc, g, name, ins[j], None, nxt)                              # masked by t_j > 0
            g = nxt
        dsc1, name1 = self._desc(B, res, n_in, h, ks[0], 1), pre + "res_path/conv_1"
        self._conv_wgrad(dsc1, sv["a"], g, name1)
        if n_in == n_out:
            self._conv_dgrad(dsc1, g, name1, x, dy, dy)                                    # in place: + d(id) = dy
            return dy
        dsc_id = self._desc(B, res, n_in, n_out, 1, 1)
        self._conv_wgrad(dsc_id, x, dy, pre + "id_path")
        dx = self._scratch(x.shape, (g, dy))
        self._conv_dgrad(dsc_id, dy, pre + "id_path", None, None, dx)
        self._conv_dgrad(dsc1, g, name1, x, dx, dx)
        return dx

    def backward(self, grad_scale=1.0, on_bucket_ready=None):
        """Back-propagates d(loss); gradients ACCUMULATE into self.grads.  on_bucket_ready(start, end) announces the
        decoder (+ the aux slots behind it) as soon as the decoder's input projection is done, then the encoder."""
        b = self._b
        B = self._img.shape[0]
        rows = B * self.hw * self.hw
        if grad_scale != 1.0:
            raise L.DB200Error("PaperVaeEngine.backward: fold grad_scale into the Adam step (grad_scale argument there)")
        dx = self._to_act(b["drecon"], b["drecon_act"])
        d1 = self._desc(B, self.H, self.dec_out_cin, self.out_C, 1, 1)
        ops.conv2d_wgrad(d1, b["dec_relu"], dx, self.G("decoder/output/conv/kernel"), self.G("decoder/output/conv/bias"))
        g = self._scratch(self._dec_last.shape)
        ops.conv2d_dgrad(d1, dx, self.P("decoder/output/conv/kernel"), self._dec_last, None, g)   # ReLU backward
        dx = g
        inputs = [self._z] + [sv.get("up", sv["y"]) for sv in b["dec"][:-1]]
        for blk, sv, x_in in reversed(list(zip(self.dec, b["dec"], inputs))):
            if blk[5] == "up":
                low = self._scratch(sv["y"].shape, (dx,))
                dx = ops.upsample2x_bwd(dx, low)
            dx = self._block_bwd(B, blk, x_in, sv, dx)
        # decoder input projection: its gradients and d(loss)/d(y_out) for the quantiser
        gk, gb = self.G("decoder/input/kernel").view(self.K, self.n_init), self.G("decoder/input/bias")
        if self.use_bf16:
            dz = dx.view(rows, self.n_init)                                                       # exactly bf16
            ops.linear_wgrad(b["y_hi"], dz, gk); ops.linear_wgrad(b["y_lo"], dz, gk)
            ops.colsum(dz, gb)
            ops.gemm(dz, self.di_hi, b["dy"], rows, self.K, self.n_init, a_mn=False, b_mn=False)
            ops.gemm(dz, self.di_lo, b["dy"], rows, self.K, self.n_init, a_mn=False, b_mn=False, mode=L.EPI_ATOMIC,
                     split_k=1)
        else:
            dsc = self._desc(B, self.hw, self.K, self.n_init, 1, 1)
            ops.conv2d_wgrad(dsc, b["y_out"], dx, self.G("decoder/input/kernel"), gb)
            ops.conv2d_dgrad(dsc, dx, self.P("decoder/input/kernel"), None, None, b["dy"])
        if on_bucket_ready:
            s0, _ = self.layout.span("decoder/input/kernel", "decoder/input/kernel")
            _, e0 = self.layout.span("decoder/output/conv/bias", "decoder/output/conv/bias")
            on_bucket_ready(s0, e0 + 64)      # + the aux scalars behind the last parameter
        self._gumbel_backward(rows)
        # encoder output projection
        gk, gb = self.G("encoder/output/conv/kernel").view(self.n_hid, self.K), self.G("encoder/output/conv/bias")
        if self.use_bf16:
            ops.split_f32(b["dlogits"], b["dl_hi"], b["dl_lo"])
            a = b["enc_relu"].view(rows, self.n_hid)
            ops.linear_wgrad(a, b["dl_hi"], gk); ops.linear_wgrad(a, b["dl_lo"], gk)
            ops.colsum(b["dl_hi"], gb); ops.colsum(b["dl_lo"], gb)
            for i, (dl, w) in enumerate(((b["dl_hi"], self.eo_hi), (b["dl_hi"], self.eo_lo), (b["dl_lo"], self.eo_hi))):
                ops.gemm(dl, w, b["denc_f32"], rows, self.n_hid, self.K, a_mn=False, b_mn=False,
                         mode=L.EPI_ATOMIC if i else L.EPI_STORE, split_k=1)
            dx = self._scratch(self._enc_last.shape)
            ops.cast_f32_to_bf16(b["denc_f32"], dx)
            ops.residual_gain(dx, 1.0, mask=self._enc_last, y=dx)                                 # ReLU backward
        else:
            dsc = self._desc(B, self.hw, self.n_hid, self.K, 1, 1)
            ops.conv2d_wgrad(dsc, b["enc_relu"], b["dlogits"], self.G("encoder/output/conv/kernel"), gb)
            dx = self._scratch(self._enc_last.shape)
            ops.conv2d_dgrad(dsc, b["dlogits"], self.P("encoder/output/conv/kernel"), self._enc_last, None, dx)
        inputs = [b["x0"]] + [sv.get("pool", sv["y"]) for sv in b["enc"][:-1]]
        for blk, sv, x_in in reversed(list(zip(self.enc, b["enc"], inputs))):
            if blk[5] == "pool":
                full = self._scratch(sv["y"].shape, (dx,))
                dx = ops.maxpool2x2_bwd(sv["y"], dx, full)
            dx = self._block_bwd(B, blk, x_in, sv, dx)
        ops.conv7x7_in_wgrad(self._img_in, dx, self.G("encoder/input/kernel"), self.G("encoder/input/bias"))
        if on_bucket_ready:
            on_bucket_ready(*self.layout.span("encoder/input/kernel", "encoder/output/conv/bias"))
