"""DALL-E transformer training engine on the sm_90a kernels (host side: buffer plan + kernel sequencing).

Mirrors what the reference builds as an mtf graph in src/dalle_mtf/models.py:141-416 and differentiates with
mtf.gradients (src/optimizers.py:34): here forward and backward are explicit kernel sequences over pre-allocated
buffers.  PyTorch owns the memory; all arithmetic is in libdalle_b200.so.

HBM layout
  * parameters, gradients, Adam m / v: ONE flat fp32 buffer each, same offsets (``ParamLayout``), plus a flat bf16
    "shadow" copy of the parameters that the GEMMs / gather read (mtf VariableDType: slice fp32 -> activation bf16,
    src/dalle_mtf/ops.py:76-82).  Order = forward order, so backward finishes gradients from the END of the buffer
    towards the front and contiguous tail ranges can be all-reduced while backward is still running.
  * q|k|v kernels are stored fused as one [d, 3d] matrix (columns q, k, v), the vocabulary projection as
    [d, Vpad] with Vpad = V rounded up to 64 (TMA needs 16-byte row pitch; pad columns stay exactly zero).
  * activations bf16 [T = B*S, features]; per-layer intermediates are kept for backward unless recompute_grad.
"""
import math

import torch

from . import lib as L
from . import ops

BF16, F32, I32 = torch.bfloat16, torch.float32, torch.int32


def _round_up(x, m):
    return (x + m - 1) // m * m


class ParamLayout:
    """name -> (offset, shape) inside the flat buffers.  Every offset is a multiple of 64 elements."""

    def __init__(self):
        self.entries = {}
        self.order = []
        self.size = 0

    def add(self, name, shape):
        n = 1
        for s in shape:
            n *= s
        self.entries[name] = (self.size, tuple(shape))
        self.order.append(name)
        self.size += _round_up(n, 64)

    def view(self, flat, name):
        off, shape = self.entries[name]
        n = 1
        for s in shape:
            n *= s
        return flat[off:off + n].view(*shape)

    def span(self, first, last):
        """[start, end) element range covering entries first..last (inclusive, in layout order)."""
        o0, _ = self.entries[first]
        o1, shp = self.entries[last]
        n = 1
        for s in shp:
            n *= s
        return o0, o1 + _round_up(n, 64)


class DalleEngine:
    """One data-parallel replica of the DALL-E decoder (src/dalle_mtf/models.py:141-416)."""

    VECTOR_PARAMS = ("ln1_g", "ln1_b", "o_b", "ln2_g", "ln2_b", "b1", "b2", "lnf_g", "lnf_b", "bout")

    def __init__(self, n_embd, n_layers, n_heads, text_vocab_size, image_vocab_size, text_seq_len, image_seq_len,
                 device="cuda", recompute_grad=False, attn_scale=1.0, ln_eps=1e-5, zero=None):
        """zero: a DataParallel with world > 1 turns on optimiser-state sharding (ZeRO-1, SURVEY.md §7 "12 B in pure
        DP"): fp32 master / Adam m / Adam v exist only for this rank's 1/N slice of the flat buffer, the bf16 compute
        copy and the fp32 gradients stay full; after the (all-reduced) gradients are final every rank updates its
        slice and the bf16 parameters are all-gathered in place.  Still data parallel: same batch split, same maths."""
        L.require_device()
        self.d, self.L, self.H = n_embd, n_layers, n_heads
        assert n_embd % n_heads == 0, "n_state must be divisible by n_heads"  # src/dalle_mtf/models.py:232
        self.dh = n_embd // n_heads
        if self.dh not in (64, 128):
            raise L.DB200Error(f"head_dim {self.dh} unsupported by the attention kernels (64 or 128)")
        if n_embd % 256 != 0:
            raise L.DB200Error(f"n_embd {n_embd} must be a multiple of 256 (LayerNorm kernels)")
        self.text_vocab_size, self.image_vocab_size = text_vocab_size, image_vocab_size
        self.text_seq_len, self.image_seq_len = text_seq_len, image_seq_len
        self.S = text_seq_len + image_seq_len                       # models.py:153
        self.V = text_vocab_size + image_vocab_size + 1             # models.py:157 (extra id = EOS)
        self.eos_token_id = self.V - 1                              # models.py:158
        self.Vpad = _round_up(self.V, 64)
        self.device = torch.device(device)
        self.recompute_grad = bool(recompute_grad)
        self.attn_scale = float(attn_scale)
        self.ln_eps = float(ln_eps)

        d, V, S, Lyr = self.d, self.V, self.S, self.L
        lay = ParamLayout()
        lay.add("wte", (V, d))
        lay.add("wpe", (S, d))
        for i in range(Lyr):
            p = f"l{i}."
            lay.add(p + "ln1_g", (d,)); lay.add(p + "ln1_b", (d,))
            lay.add(p + "wqkv", (d, 3 * d))
            lay.add(p + "wo", (d, d)); lay.add(p + "o_b", (d,))
            lay.add(p + "ln2_g", (d,)); lay.add(p + "ln2_b", (d,))
            lay.add(p + "w1", (d, 4 * d)); lay.add(p + "b1", (4 * d,))
            lay.add(p + "w2", (4 * d, d)); lay.add(p + "b2", (d,))
        lay.add("lnf_g", (d,)); lay.add("lnf_b", (d,))
        lay.add("wout", (d, self.Vpad)); lay.add("bout", (self.Vpad,))
        self.layout = lay
        self.n_params_padded = lay.size
        # trailing 64 floats of the gradient buffer carry scalars that ride along with the gradient all-reduce:
        #   [0] = sum of per-token losses of this rank / (global tokens)
        self.aux_off = lay.size
        n = lay.size + 64
        dev = self.device
        self._views = {}
        self.zero = zero if (zero is not None and getattr(zero, "world", 1) > 1) else None
        self.grads = torch.zeros(n, dtype=F32, device=dev)
        if self.zero is None:
            self.master = torch.zeros(n, dtype=F32, device=dev)
            self.adam_m = torch.zeros(n, dtype=F32, device=dev)
            self.adam_v = torch.zeros(n, dtype=F32, device=dev)
            self.shadow = torch.zeros(n, dtype=BF16, device=dev)
            self.shard = (0, lay.size)
        else:
            w, r = self.zero.world, self.zero.rank
            self.chunk = _round_up(-(-lay.size // w), 64)                 # elements per rank (equal: in-place all-gather)
            self.shard = (min(r * self.chunk, lay.size), min((r + 1) * self.chunk, lay.size))
            self.master = torch.zeros(self.chunk, dtype=F32, device=dev)  # this rank's slice only
            self.adam_m = torch.zeros(self.chunk, dtype=F32, device=dev)
            self.adam_v = torch.zeros(self.chunk, dtype=F32, device=dev)
            self.shadow = torch.zeros(max(w * self.chunk, n), dtype=BF16, device=dev)
            # compact fp32 copy of the vector parameters (LayerNorm g / b, biases) the kernels read in fp32: rebuilt
            # from the bf16 parameters after every all-gather — mtf casts every variable to the activation dtype when
            # it is used (src/dalle_mtf/ops.py:76-82), so this is the reference's own bf16 policy
            self._vec_off, table, off = {}, [], 0
            for name in lay.order:
                if name.split(".")[-1] in self.VECTOR_PARAMS:
                    o, shp = lay.entries[name]
                    self._vec_off[name] = (off, shp)
                    table += [o, off, shp[0]]
                    off += _round_up(shp[0], 64)
            self.vec32 = torch.zeros(off, dtype=F32, device=dev)
            self._vec_table = torch.tensor(table, dtype=torch.int64, device=dev)
        self.gnorm_sq = torch.zeros(1, dtype=F32, device=dev)
        self._grads_clean = False
        self._bufs = None
        self._buf_key = None

    # ------------------------------------------------------------------------------------------ parameters
    # The flat buffers are allocated once and only ever written in place, so the per-name views are cached: building a
    # slice + view costs a few microseconds of host time, and the decode loop asks for ~70 of them per position.
    def _view(self, which, flat, name):
        key = (which, name)
        v = self._views.get(key)
        if v is None:
            v = self._views[key] = self.layout.view(flat, name)
        return v

    def P(self, name):  # fp32 view of a parameter (ZeRO-1: only the vector parameters exist in full fp32)
        if self.zero is not None:
            if name not in self._vec_off:
                raise L.DB200Error(f"{name}: the fp32 master of a matrix is sharded across ranks in ZeRO-1 mode")
            key = (3, name)
            v = self._views.get(key)
            if v is None:
                off, shp = self._vec_off[name]
                v = self._views[key] = self.vec32[off:off + shp[0]]
            return v
        return self._view(0, self.master, name)

    def W(self, name):  # bf16 compute copy
        return self._view(1, self.shadow, name)

    def G(self, name):  # fp32 gradient view
        return self._view(2, self.grads, name)

    def n_params(self):
        """Trainable parameter count as the reference would print it (src/utils/utils.py:55-70)."""
        d, V, S, Lyr = self.d, self.V, self.S, self.L
        return V * d + S * d + Lyr * (2 * d + 3 * d * d + d * d + d + 2 * d + 4 * d * d + 4 * d + 4 * d * d + d) + \
            2 * d + d * V + V

    @staticmethod
    def _ref_names(i):
        pre = f"layer_{i}/"
        return {
            "ln1_g": pre + "norm_1/g", "ln1_b": pre + "norm_1/b", "wo": pre + "attn/o",
            "o_b": pre + "attn/compute_output_bias/o_b", "ln2_g": pre + "norm_2/g", "ln2_b": pre + "norm_2/b",
            "w1": pre + "mlp/mlp_linear_1/kernel", "b1": pre + "mlp/mlp_linear_1/bias",
            "w2": pre + "mlp/mlp_linear_2/kernel", "b2": pre + "mlp/mlp_linear_2/bias",
        }

    def load_params(self, named):
        """Load a dict keyed by the reference's variable names (SURVEY.md Appendix B); CPU or CUDA fp32 tensors."""
        self.load_flat(self.master, named)
        self.refresh_shadow()

    def _scatter_full(self, name, t, cols=None):
        """ZeRO-1: place a full fp32 parameter tensor: bf16 copy (full) + the part of it inside this rank's slice."""
        off, shape = self.layout.entries[name]
        dst16 = self.layout.view(self.shadow, name)
        if cols is not None:
            dst16 = dst16[:, :cols] if dst16.dim() == 2 else dst16[:cols]
        dst16.copy_(t)
        full = torch.zeros(shape, dtype=F32, device=self.device)
        (full[:, :cols] if (cols is not None and full.dim() == 2) else (full[:cols] if cols is not None else full)).copy_(t)
        lo, hi = self.shard
        n = full.numel()
        a, b = max(lo, off), min(hi, off + n)
        if a < b:
            self.master[a - lo:b - lo].copy_(full.view(-1)[a - off:b - off])

    def _refresh_vecs(self):
        ops.gather_cast(self.shadow, self.vec32, self._vec_table, self._vec_table.numel() // 3)

    def load_flat(self, flat, named):
        """Fill one of the flat fp32 buffers (master | adam_m | adam_v) from a dict of reference-named tensors."""
        dev = self.device
        if self.zero is not None:
            if flat is not self.master:
                raise L.DB200Error("ZeRO-1 mode: loading sharded Adam slots is not implemented (throughput configuration)")
            self.master.zero_(); self.shadow.zero_()
            f32 = lambda x: x.to(device=dev, dtype=F32)
            self._scatter_full("wte", f32(named["embedding/wte"]))
            self._scatter_full("wpe", f32(named["positional_embedding/wpe"]))
            for i in range(self.L):
                p = f"l{i}."
                for k, rn in self._ref_names(i).items():
                    self._scatter_full(p + k, f32(named[rn]))
                pre = f"layer_{i}/attn/"
                self._scatter_full(p + "wqkv", torch.cat([f32(named[pre + "q"]), f32(named[pre + "k"]),
                                                          f32(named[pre + "v"])], dim=1))
            self._scatter_full("lnf_g", f32(named["to_logits/layer_norm/g"]))
            self._scatter_full("lnf_b", f32(named["to_logits/layer_norm/b"]))
            self._scatter_full("wout", f32(named["to_logits/linear_out/kernel"]), cols=self.V)
            self._scatter_full("bout", f32(named["to_logits/linear_out/bias"]), cols=self.V)
            self._refresh_vecs()
            return
        flat.zero_()
        view = lambda n: self.layout.view(flat, n)

        def put(name, t):
            dst = view(name)
            t = t.to(device=dev, dtype=F32)
            if tuple(t.shape) != tuple(dst.shape):
                raise L.DB200Error(f"load_params: {name}: expected {tuple(dst.shape)}, got {tuple(t.shape)}")
            dst.copy_(t)

        put("wte", named["embedding/wte"])
        put("wpe", named["positional_embedding/wpe"])
        for i in range(self.L):
            p = f"l{i}."
            ref = self._ref_names(i)
            for k, rn in ref.items():
                put(p + k, named[rn])
            pre = f"layer_{i}/attn/"
            put(p + "wqkv", torch.cat([named[pre + "q"], named[pre + "k"], named[pre + "v"]], dim=1))
        put("lnf_g", named["to_logits/layer_norm/g"]); put("lnf_b", named["to_logits/layer_norm/b"])
        view("wout")[:, :self.V].copy_(named["to_logits/linear_out/kernel"].to(device=dev, dtype=F32))
        view("bout")[:self.V].copy_(named["to_logits/linear_out/bias"].to(device=dev, dtype=F32))

    def export_params(self, source=None):
        """Inverse of load_params: dict of reference-named fp32 CPU tensors (source: master | grads | adam_m | adam_v).
        ZeRO-1: parameters are exported from the full bf16 copy (the reference checkpoints bf16 "master" values under
        bf_16 too, src/dalle_mtf/ops.py:79-80); the sharded Adam slots cannot be exported from one rank."""
        if self.zero is not None and (source is None or source is self.master):
            source = self.shadow
        elif self.zero is not None and source is not self.grads:
            raise L.DB200Error("ZeRO-1 mode: the Adam slots are sharded across ranks")
        flat = self.master if source is None else source
        view = lambda n: self.layout.view(flat, n).detach().float().cpu().clone()
        out = {"embedding/wte": view("wte"), "positional_embedding/wpe": view("wpe")}
        d = self.d
        for i in range(self.L):
            p = f"l{i}."
            for k, rn in self._ref_names(i).items():
                out[rn] = view(p + k)
            wqkv = view(p + "wqkv")
            pre = f"layer_{i}/attn/"
            out[pre + "q"], out[pre + "k"], out[pre + "v"] = wqkv[:, :d].clone(), wqkv[:, d:2 * d].clone(), \
                wqkv[:, 2 * d:].clone()
        out["to_logits/layer_norm/g"], out["to_logits/layer_norm/b"] = view("lnf_g"), view("lnf_b")
        out["to_logits/linear_out/kernel"] = view("wout")[:, :self.V].clone()
        out["to_logits/linear_out/bias"] = view("bout")[:self.V].clone()
        return out

    def init_params(self, seed=0):
        """Reference initialisers (SURVEY.md Appendix B), drawn on the device; identical on every rank for a seed."""
        g = torch.Generator(device=self.device).manual_seed(seed)
        d, H, dh, Lyr = self.d, self.H, self.dh, self.L
        if self.zero is not None:
            return self._init_params_sharded(g)
        self.master.zero_()

        def normal(name, std, cols=None):
            t = self.P(name)
            if cols is not None:
                t = t[:, :cols] if t.dim() == 2 else t[:cols]
            t.copy_(torch.randn(t.shape, generator=g, device=self.device, dtype=F32) * std)

        normal("wte", 0.02); normal("wpe", 0.01)
        for i in range(Lyr):
            p = f"l{i}."
            self.P(p + "ln1_g").fill_(1.0); self.P(p + "ln2_g").fill_(1.0)
            wqkv = self.P(p + "wqkv")
            wqkv[:, :d].copy_(torch.randn(d, d, generator=g, device=self.device) * (d ** -0.5 * dh ** -0.5))
            wqkv[:, d:].copy_(torch.randn(d, 2 * d, generator=g, device=self.device) * (d ** -0.5))
            normal(p + "wo", (H * dh) ** -0.5)
            normal(p + "w1", 0.02)
            normal(p + "w2", 0.02 / math.sqrt(Lyr))
        self.P("lnf_g").fill_(1.0)
        normal("wout", 0.02, cols=self.V)
        self.refresh_shadow()

    def _init_params_sharded(self, g):
        """Same initialisers and the same random stream as init_params, one tensor at a time (ZeRO-1: no full fp32 buffer)."""
        d, H, dh, Lyr = self.d, self.H, self.dh, self.L
        self.master.zero_(); self.shadow.zero_()
        rn = lambda shape, std: torch.randn(shape, generator=g, device=self.device, dtype=F32) * std
        ones = lambda n: torch.ones(n, dtype=F32, device=self.device)
        self._scatter_full("wte", rn((self.V, d), 0.02)); self._scatter_full("wpe", rn((self.S, d), 0.01))
        for i in range(Lyr):
            p = f"l{i}."
            self._scatter_full(p + "ln1_g", ones(d)); self._scatter_full(p + "ln2_g", ones(d))
            wq = torch.randn(d, d, generator=g, device=self.device) * (d ** -0.5 * dh ** -0.5)
            wkv = torch.randn(d, 2 * d, generator=g, device=self.device) * (d ** -0.5)
            self._scatter_full(p + "wqkv", torch.cat([wq, wkv], dim=1))
            self._scatter_full(p + "wo", rn((d, d), (H * dh) ** -0.5))
            self._scatter_full(p + "w1", rn((d, 4 * d), 0.02))
            self._scatter_full(p + "w2", rn((4 * d, d), 0.02 / math.sqrt(Lyr)))
        self._scatter_full("lnf_g", ones(d))
        self._scatter_full("wout", rn((d, self.V), 0.02), cols=self.V)
        self._refresh_vecs()

    def refresh_shadow(self):
        if self.zero is not None:
            return self._refresh_vecs()
        ops.cast_f32_to_bf16(self.master[:self.n_params_padded], self.shadow[:self.n_params_padded])

    # ------------------------------------------------------------------------------------------ buffers
    def _alloc(self, B):
        key = (B,)
        if self._buf_key == key:
            return self._bufs
        dev, d, S, T = self.device, self.d, self.S, B * self.S
        e = lambda *shape, dtype=BF16: torch.empty(*shape, dtype=dtype, device=dev)
        nt = ops.ce_tiles(self.Vpad)
        n_saved = 1 if self.recompute_grad else self.L
        b = {
            "xs": [e(T, d) for _ in range(self.L + 1)],        # residual stream at every layer boundary
            "layers": [{
                "ln1": e(T, d), "mean1": e(T, dtype=F32), "rstd1": e(T, dtype=F32),
                "qkv": e(T, 3 * d), "attn": e(T, d), "lse": e(B, self.H, S, dtype=F32),
                "xmid": e(T, d), "ln2": e(T, d), "mean2": e(T, dtype=F32), "rstd2": e(T, dtype=F32),
                "h1": e(T, 4 * d),
            } for _ in range(n_saved)],
            "hf": e(T, d), "meanf": e(T, dtype=F32), "rstdf": e(T, dtype=F32),
            "labels": e(B, S, dtype=I32),
            "part_max": e(nt, T, dtype=F32), "part_sum": e(nt, T, dtype=F32),
            "label_logit": e(T, dtype=F32), "lse_v": e(T, dtype=F32), "loss_rows": e(T, dtype=F32),
            "dlogits": e(T, self.Vpad),
            # backward scratch
            "dx_a": e(T, d), "dx_b": e(T, d), "dtmp": e(T, d), "dh1": e(T, 4 * d), "dqkv": e(T, 3 * d),
            "delta": e(B, self.H, S, dtype=F32), "dq_acc": e(1, dtype=F32),
        }
        self._bufs, self._buf_key = b, key
        return b

    # ------------------------------------------------------------------------------------------ forward
    def _block_fwd(self, i, x_in, x_out, sv, B):
        """DALLE.block (src/dalle_mtf/models.py:326-335): x += attn(LN1 x); x += mlp(LN2 x)."""
        p = f"l{i}."
        ops.layernorm_fwd(x_in, self.P(p + "ln1_g"), self.P(p + "ln1_b"), sv["ln1"], sv["mean1"], sv["rstd1"],
                          self.ln_eps)
        ops.linear_fwd(sv["ln1"], self.W(p + "wqkv"), sv["qkv"])                       # q|k|v, no bias (:242-244)
        ops.attn_fwd(sv["qkv"], sv["attn"], sv["lse"], B, self.S, self.H, self.dh, self.attn_scale)
        ops.linear_fwd(sv["attn"], self.W(p + "wo"), sv["xmid"], bias=self.P(p + "o_b"), residual=x_in)  # :303-311,330
        ops.layernorm_fwd(sv["xmid"], self.P(p + "ln2_g"), self.P(p + "ln2_b"), sv["ln2"], sv["mean2"], sv["rstd2"],
                          self.ln_eps)
        ops.linear_fwd(sv["ln2"], self.W(p + "w1"), sv["h1"], bias=self.P(p + "b1"), relu=True)     # :320
        ops.linear_fwd(sv["h1"], self.W(p + "w2"), x_out, bias=self.P(p + "b2"), residual=sv["xmid"])  # :321,333

    def forward(self, tokens, loss_accum=None):
        """tokens int32 [B,S] on the device.  Adds sum_t loss_rows[t] of this batch into the 1-element fp32 tensor
        `loss_accum` (default: the aux slot behind the gradients, which rides along with the gradient all-reduce)
        and returns it.  The mean over all positions (src/dalle_mtf/models.py:353-354) is that sum / (global B*S)."""
        B, S = tokens.shape
        assert S == self.S, f"expected sequence length {self.S}, got {S}"
        bufs = self._alloc(B)
        T = B * S
        self._tokens = tokens
        ops.embed_fwd(tokens, self.W("wte"), self.W("wpe"), bufs["xs"][0].view(B, S, self.d))    # models.py:399
        for i in range(self.L):
            sv = bufs["layers"][0 if self.recompute_grad else i]
            self._block_fwd(i, bufs["xs"][i], bufs["xs"][i + 1], sv, B)
        ops.layernorm_fwd(bufs["xs"][self.L], self.P("lnf_g"), self.P("lnf_b"), bufs["hf"], bufs["meanf"],
                          bufs["rstdf"], self.ln_eps)                                            # models.py:393
        ops.shift_labels(tokens, bufs["labels"], self.eos_token_id)                                # models.py:407-410
        labels = bufs["labels"].view(T)
        ops.gemm(bufs["hf"], self.W("wout"), None, T, self.Vpad, self.d, a_mn=False, b_mn=True, mode=L.EPI_CE_STATS,
                 bias=self.P("bout"), labels=labels, part_max=bufs["part_max"], part_sum=bufs["part_sum"],
                 label_logit=bufs["label_logit"], n_valid=self.V)
        if loss_accum is None:
            loss_accum = self.grads[self.aux_off:self.aux_off + 1]
        ops.ce_finish(bufs["part_max"], bufs["part_sum"], bufs["label_logit"], bufs["lse_v"], bufs["loss_rows"],
                      loss_accum)
        return loss_accum

    def logits(self, tokens):
        """fp32 logits [B,S,V] (return_logits=True path, src/dalle_mtf/models.py:412-415).  Test / eval use only:
        this materialises the tensor the training path never writes."""
        B, S = tokens.shape
        self.forward(tokens, loss_accum=torch.zeros(1, dtype=F32, device=self.device))
        T = B * S
        out = torch.empty(T, self.Vpad, dtype=F32, device=self.device)
        ops.gemm(self._bufs["hf"], self.W("wout"), out, T, self.Vpad, self.d, a_mn=False, b_mn=True,
                 bias=self.P("bout"))
        return out.view(B, S, self.Vpad)[:, :, :self.V]

    # ------------------------------------------------------------------------------------------ backward
    def _block_bwd(self, i, x_in, sv, dx_out, dx_in, bufs, B, dxsum_below):
        """Backward of one block.  Bias gradients are column sums of activation gradients; they are produced by the
        kernel that WRITES that gradient (LayerNorm-backward / ReLU-mask epilogue) instead of separate passes:
        db2 (= colsum of this block's output gradient) was already accumulated by whoever produced dx_out."""
        p = f"l{i}."
        # ---- MLP
        ops.linear_dgrad(dx_out, self.W(p + "w2"), bufs["dh1"], relu_mask_of=sv["h1"],
                         colsum=self.G(p + "b1"))                                       # dH = (dx W2^T)*[h1>0]; db1
        ops.linear_wgrad(sv["h1"], dx_out, self.G(p + "w2"))
        ops.linear_dgrad(bufs["dh1"], self.W(p + "w1"), bufs["dtmp"])                         # dLN2 out
        ops.linear_wgrad(sv["ln2"], bufs["dh1"], self.G(p + "w1"))
        dx_mid = bufs["dx_b"] if dx_out is bufs["dx_a"] else bufs["dx_a"]
        ops.layernorm_bwd(bufs["dtmp"], sv["xmid"], self.P(p + "ln2_g"), sv["mean2"], sv["rstd2"], dx_out, dx_mid,
                          self.G(p + "ln2_g"), self.G(p + "ln2_b"), dxsum=self.G(p + "o_b"))  # do_b = colsum(dx_mid)
        # ---- attention
        ops.linear_dgrad(dx_mid, self.W(p + "wo"), bufs["dtmp"])                              # d(attn out)
        ops.linear_wgrad(sv["attn"], dx_mid, self.G(p + "wo"))
        ops.attn_bwd(sv["qkv"], sv["attn"], bufs["dtmp"], sv["lse"], bufs["dq_acc"], bufs["delta"], bufs["dqkv"], B,
                     self.S, self.H, self.dh, self.attn_scale)
        ops.linear_dgrad(bufs["dqkv"], self.W(p + "wqkv"), bufs["dtmp"])                      # dLN1 out
        ops.linear_wgrad(sv["ln1"], bufs["dqkv"], self.G(p + "wqkv"))
        ops.layernorm_bwd(bufs["dtmp"], x_in, self.P(p + "ln1_g"), sv["mean1"], sv["rstd1"], dx_mid, dx_in,
                          self.G(p + "ln1_g"), self.G(p + "ln1_b"), dxsum=dxsum_below)        # db2 of the layer below

    def backward(self, grad_scale, on_bucket_ready=None):
        """Back-propagates d(sum(loss_rows) * grad_scale).  Gradients ACCUMULATE into self.grads.
        on_bucket_ready(start, end) is called as soon as the flat range [start, end) is final (data-parallel hook)."""
        bufs = self._bufs
        tokens = self._tokens
        B, S = tokens.shape
        T, d = B * S, self.d
        labels = bufs["labels"].view(T)
        ops.gemm(bufs["hf"], self.W("wout"), bufs["dlogits"], T, self.Vpad, d, a_mn=False, b_mn=True,
                 mode=L.EPI_CE_GRAD, alpha=grad_scale, bias=self.P("bout"), labels=labels, lse=bufs["lse_v"],
                 n_valid=self.V, colsum=self.G("bout"))                 # dlogits + fused d(bout) = colsum(dlogits)
        ops.linear_wgrad(bufs["hf"], bufs["dlogits"], self.G("wout"))
        ops.linear_dgrad(bufs["dlogits"], self.W("wout"), bufs["dtmp"])
        dx = bufs["dx_a"]
        ops.layernorm_bwd(bufs["dtmp"], bufs["xs"][self.L], self.P("lnf_g"), bufs["meanf"], bufs["rstdf"], None, dx,
                          self.G("lnf_g"), self.G("lnf_b"), dxsum=self.G(f"l{self.L - 1}.b2"))   # db2 of the last block
        if on_bucket_ready:
            s, e = self.layout.span("lnf_g", "bout")
            on_bucket_ready(s, e + 64)  # + the aux scalars (loss) that sit behind the last parameter
        for i in reversed(range(self.L)):
            if self.recompute_grad:  # mtf.recompute_grad per block, src/dalle_mtf/models.py:342-343
                sv = bufs["layers"][0]
                self._block_fwd(i, bufs["xs"][i], bufs["dtmp"], sv, B)
            else:
                sv = bufs["layers"][i]
            # dx (grad w.r.t. the block output) is dead once dx_mid has been formed in the other buffer, so the
            # block's input gradient is written back into the same storage.
            self._block_bwd(i, bufs["xs"][i], sv, dx, dx, bufs, B, self.G(f"l{i - 1}.b2") if i > 0 else None)
            if on_bucket_ready:
                s, e = self.layout.span(f"l{i}.ln1_g", f"l{i}.b2")
                on_bucket_ready(s, e)
        ops.embed_bwd(tokens, dx.view(B, S, d), self.G("wte"), self.G("wpe"))
        if on_bucket_ready:
            s, e = self.layout.span("wte", "wpe")
            on_bucket_ready(s, e)

    # ------------------------------------------------------------------------------------------ optimiser
    def zero_grads(self):
        """Gradients accumulate (+=), so every step starts from zeros.  The Adam kernel writes those zeros while it
        streams the gradient it consumes, so after an optimiser step only the 64 aux scalars (loss) need clearing; the
        full 4 B/param memset runs only when backward ran without an optimiser step in between (tests, first step)."""
        if self._grads_clean:
            self.grads[self.aux_off:].zero_()
        else:
            self.grads.zero_()
        self._grads_clean = False

    def _decay_segments(self):
        """Contiguous [start, end, decays) runs of the flat buffer: mtf's AdamWeightDecayOptimizer is built with
        exclude_from_weight_decay=["norm", "bias"] (src/optimizers.py:84-88), i.e. every variable whose NAME contains
        "norm" or "bias" (LayerNorm g/b, all biases incl. compute_output_bias/o_b) is left undecayed."""
        if getattr(self, "_segs", None) is None:
            decays = lambda n: n in ("wte", "wpe", "wout") or n.split(".")[-1] in ("wqkv", "wo", "w1", "w2")
            segs = []
            for name in self.layout.order:
                s, e = self.layout.span(name, name)
                d = decays(name)
                if segs and segs[-1][2] == d and segs[-1][1] == s:
                    segs[-1][1] = e
                else:
                    segs.append([s, e, d])
            self._segs = [tuple(x) for x in segs]
        return self._segs

    def optimizer_step(self, lr, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.0, clip=1.0):
        """clip_by_global_norm + mtf AdamWeightDecayOptimizer (src/optimizers.py:11-16, 82-103); no host sync.
        clip=None disables clipping (explicit `"gradient_clipping": null`, optimizers.py:101)."""
        n = self.n_params_padded
        if clip and clip > 0:
            self.gnorm_sq.zero_()
            ops.sqnorm(self.grads[:n], self.gnorm_sq)       # the reduced gradient is identical on every rank
            gn = self.gnorm_sq
        else:
            gn, clip = None, 0.0
        if self.zero is not None:
            if weight_decay:
                raise L.DB200Error("ZeRO-1 mode: weight_decay != 0 is not wired (no reference config uses it)")
            lo, hi = self.shard
            m = hi - lo
            if m > 0:   # this rank's slice: fp32 master + Adam slots, bf16 result written into the full copy
                ops.adam_step(self.master[:m], self.adam_m[:m], self.adam_v[:m], self.grads[lo:hi], self.shadow[lo:hi],
                              lr, beta1, beta2, eps, 0.0, gn, clip, 1.0, False, 0)
            self.zero.all_gather_inplace(self.shadow, self.chunk)   # bf16 parameters of every slice
            self._refresh_vecs()
            return
        if not weight_decay:
            ops.adam_step(self.master[:n], self.adam_m[:n], self.adam_v[:n], self.grads[:n], self.shadow[:n], lr,
                          beta1, beta2, eps, 0.0, gn, clip, 1.0, False, 0, zero_grad=True)
            self._grads_clean = True
            return
        for s, e, d in self._decay_segments():     # `update += weight_decay * param` only on the kernels / embeddings
            ops.adam_step(self.master[s:e], self.adam_m[s:e], self.adam_v[s:e], self.grads[s:e], self.shadow[s:e], lr,
                          beta1, beta2, eps, weight_decay if d else 0.0, gn, clip, 1.0, False, 0)
