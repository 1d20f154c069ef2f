"""Autoregressive sampling with a K/V cache ("next" row N4, SURVEY.md §8f).

The reference only sketches this path: `DALLE(is_incremental_inference=True, context=...)` blends the current
position's k, v into the cached states at `context.position - 1` and lets that position's query attend to keys up to
itself (src/dalle_mtf/models.py:246-254, 281-285); PREDICT mode raises NotImplementedError (src/model_fns.py:135-136)
and no sampling loop exists.  What is implemented here is that sketch, driven one position at a time over the SAME
parameters and the same kernels' numerics as training:

  per position p:   x = wte[token] + wpe[p]                                     (embed_fwd_at)
  per layer:        q|k|v = LN1(x) Wqkv;  cache[p] = k, v;  a = softmax_{j<=p}(q.k_j) v_j   (attn_decode;
                    a local layer of radius r takes j > p - r only, models.py:257-273; an axial layer the text
                    positions and p's image row or column; a conv layer the text positions and p's k x k window;
                    a block-sparse layer the positions <= p of the blocks its layout lets p's block see)
                    x = x + a Wo + o_b;  x = x + act(LN2(x) W1 + b1) W2 + b2   (the training GEMM, M = batch rows;
                    act = ReLU, or GELU without a pre-activation output); with rotary embeddings q and k are
                    rotated to position p (rope_decode) before k enters the cache (rotary_emb: q, k and v,
                    rope_emb_decode, before k and v enter it); with the token shift each
                    LayerNorm output's first d/2 columns enter a per-layer cache and are replaced by the shifted
                    chunks of positions p - 1 and p - W (shift_tokens_decode); with the sandwich LayerNorm each
                    branch output is normalised before its residual add (layernorm_residual_fwd); with LayerScale
                    what a branch adds is multiplied by its per-channel scale (DalleEngine.branch_add)
  logits = LN_f(x) Wout + bout (fp32), with the stable option LN_f(x / max(x)) (DalleEngine.final_ln), with a tied
           embedding LN_f(x) wte^T + bout (DalleEngine.vocab_gemm);
  next token = argmax over the allowed id range of logits / T + Gumbel noise

In generate / generate_graphed, prompt (text) positions are teacher-forced through the same step function; complete
instead runs the whole prompt (text, optionally followed by the first rows of an image's codes) through the training
forward kernels in one pass (DalleEngine.prefill) and continues from there with the same sampling step.  Image
positions are restricted to the image-token id range [image_offset, image_offset + image_vocab_size), matching the
ids training builds (src/model_fns.py:117-122; image_offset = text_vocab_size, + text_seq_len with per-position
padding).  `temperature == 0` (or None) is greedy decoding; `top_k` /
`top_p` truncate the image-token distribution (after temperature) before the Gumbel-max draw.

Classifier-free guidance (`guidance_scale` s, "condition scale"): every sampled row gets a twin whose caption is
text_seq_len padding ids (the unconditional prompt a model trained with caption dropout has learned; with
per-position padding the text_seq_len per-position pads).  The 2R rows run
through the same step kernels (R conditional rows, then R unconditional ones) and each image token is drawn once per
pair from u + s (c - u) of the two logit rows (db200_sample_rows_guided), then fed to both.  s = 1 (or None) is the
plain sampler: no twin rows, the same kernels, the same tokens.

Caption generation (generate_texts, DALLE-pytorch's generate_texts) draws the text positions instead: after a prefill
of the shortest caption prefix, each text column is drawn over the text window [0, image_offset) by the same sampling
kernels and finished by db200_caption_next (the prompt where a row's prefix is longer, padding once a padding token has
been drawn), in a third captured graph.
"""
import math
import numbers

import torch

from . import ops

BF16, F32, I32 = torch.bfloat16, torch.float32, torch.int32

# ids one filtered (top-k / top-p) draw can hold: db200_sample_rows_filtered keeps a row in one CTA's shared memory,
# SF_MAX_N = SF_SMEM_BYTES / 4 in csrc/decode.cu.  Draws without a filter, guided or not, have no such limit.
FILTER_MAX_IDS = 51200


class DalleSampler:
    def __init__(self, engine, padding_id=None):
        """padding_id: the caption id of the unconditional rows of guided sampling (default text_vocab_size - 1, the
        id GPT-2 + <|padding|> captions are padded with)."""
        self.e = engine
        pad = engine.text_vocab_size - 1 if padding_id is None else padding_id
        if isinstance(pad, bool) or int(pad) != pad or not 0 <= pad < engine.text_vocab_size:
            raise ValueError(f"padding_id must be an integer in [0, {engine.text_vocab_size}), got {padding_id!r}")
        self.padding_id = int(pad)
        self._B = None

    def _captions(self, text_ids):
        """The text positions of the prompt rows: text_ids, or with per-position padding text_ids with every padding_id
        at position p replaced by p's padding token (the training mapping, db200_assemble_tokens_pp)."""
        e = self.e
        if not e.per_position_padding:
            return text_ids
        out = torch.empty(text_ids.shape, dtype=I32, device=e.device)
        return ops.assemble_tokens_pp(text_ids.to(device=e.device, dtype=I32).contiguous(), None, out, 0,
                                      self.padding_id, e.pad_base)

    def _uncond(self, B):
        """The text positions of B unconditional (guidance) rows: padding_id everywhere, or the per-position pads."""
        if not self.e.per_position_padding:
            return self.padding_id
        return self._captions(torch.full((B, self.e.text_seq_len), self.padding_id, dtype=I32, device=self.e.device))

    def _alloc(self, B):
        if self._B == B:
            return
        self._graph_key = self._text_key = None      # captured graphs point at the buffers replaced here
        e = self.e
        dev, d = e.device, e.d
        mk = lambda *shape, dtype=BF16: torch.empty(*shape, dtype=dtype, device=dev)
        # per layer: the k / v caches, or for a gMLP layer its cache of SGU LayerNorm outputs (same bytes per token as
        # a global layer's k + v) and None
        self.kc = [mk(B, e.S, 2 * d) if e.mlp[i] else mk(B, e.S, e.H, e.dh) for i in range(e.L)]
        self.vc = [None if e.mlp[i] else mk(B, e.S, e.H, e.dh) for i in range(e.L)]
        if any(e.mlp):   # a gMLP layer's step: res | gate, gn, h
            self.g_res, self.g_gate, self.g_gn, self.g_h = mk(B, 2 * d), mk(B, 2 * d), mk(B, 2 * d), mk(B, 2 * d)
        # token shift: the unshifted first d/2 columns of every position's LN1 (2i) and LN2 (2i + 1) output of layer i
        self.sc = [mk(B, e.S, d // 2) for _ in range(2 * e.L)] if e.shift_tokens else None
        self.x = [mk(B, d), mk(B, d)]
        self.ln = mk(B, d)
        self.qkv = mk(B, 3 * d)
        self.att = mk(B, d)
        self.xmid = mk(B, d)
        self.h1 = mk(B, 4 * d)
        self.ob = mk(B, d) if e.split_branch else None    # sandwich LayerNorm / LayerScale: a branch output
        self.mean, self.rstd = mk(B, dtype=F32), mk(B, dtype=F32)
        self.mf = mk(B, dtype=F32) if e.stable else None   # stable: the DivideMax row maxima of the final LayerNorm
        self.logit = mk(B, e.Vpad, dtype=F32)
        self.tok = mk(B, dtype=I32)
        self._B = B

    def _branch_out(self, p, norm, x, w, bias, x_res, out):
        """out = x_res + x w + bias, or with the sandwich LayerNorm out = x_res + LN<norm>(x w + bias) (norm "a": the
        attention branch's LayerNorm, "m": the MLP's), what is added times s<norm> under LayerScale
        (DalleEngine.branch_add)."""
        e = self.e
        if not e.split_branch:
            return ops.linear_fwd(x, w, out, bias=bias, residual=x_res)
        ops.linear_fwd(x, w, self.ob, bias=bias)
        e.branch_add(p, norm, self.ob, x_res, out, self.mean, self.rstd)

    def _gmlp_step(self, p, i, pos=None, pos_dev=None):
        """A gMLP layer's token mixing for one position of every row, from self.ln into self.g_h: the training
        forward's two GELU products and SGU LayerNorm, then sgu_decode(_dev) over the layer's cache."""
        e, C = self.e, 2 * self.e.d
        w_in, b_in = e.W(p + "gm_win"), e.P(p + "gm_bin")
        ops.linear_fwd(self.ln, w_in[:, :C], self.g_res, bias=b_in[:C], gelu=True)
        ops.linear_fwd(self.ln, w_in[:, C:], self.g_gate, bias=b_in[C:], gelu=True)
        ops.layernorm_fwd(self.g_gate, e.P(p + "sgu_g"), e.P(p + "sgu_b"), self.g_gn, self.mean, self.rstd, e.ln_eps)
        if pos_dev is None:
            ops.sgu_decode(self.g_gn, self.g_res, e.W(p + "sgu_w"), e.P(p + "sgu_c"), self.kc[i], self.g_h, pos)
        else:
            ops.sgu_decode_dev(self.g_gn, self.g_res, e.W(p + "sgu_w"), e.P(p + "sgu_c"), self.kc[i], self.g_h,
                               pos_dev)
        return self.g_h

    def step(self, tokens_b, pos):
        """One position for every row: tokens_b int32 [B] -> fp32 logits [B, Vpad] of the NEXT position."""
        e = self.e
        ops.embed_fwd_at(tokens_b, e.embed_table(), e.pos_embedding(), self.x[0], pos)
        x_in, x_out = self.x
        for i in range(e.L):
            p = f"l{i}."
            ops.layernorm_fwd(x_in, e.P(p + "ln1_g"), e.P(p + "ln1_b"), self.ln, self.mean, self.rstd, e.ln_eps)
            if e.shift_tokens:
                ops.shift_tokens_decode(self.ln, self.sc[2 * i], pos, e.text_seq_len, e.shift_w)
            if e.mlp[i]:
                self._branch_out(p, "a", self._gmlp_step(p, i, pos=pos), e.W(p + "gm_wout"), e.P(p + "gm_bout"), x_in,
                                 self.xmid)
            else:
                ops.linear_fwd(self.ln, e.W(p + "wqkv"), self.qkv)
                if e.rotary:
                    ops.rope_decode(self.qkv, e.rope_table, pos, e.H, e.dh, e.rotary_dim)
                if e.rotary_emb:
                    ops.rope_emb_decode(self.qkv, e.rope_emb_table, pos, e.H, e.dh)
                ops.attn_decode(self.qkv, self.kc[i], self.vc[i], self.att, pos, e.attn_scale, radius=e.radii[i],
                                **e.axial_kw[i], **e.conv_kw[i], **e.block_sparse_kw[i])
                self._branch_out(p, "a", self.att, e.W(p + "wo"), e.P(p + "o_b"), x_in, self.xmid)
            ops.layernorm_fwd(self.xmid, e.P(p + "ln2_g"), e.P(p + "ln2_b"), self.ln, self.mean, self.rstd, e.ln_eps)
            if e.shift_tokens:
                ops.shift_tokens_decode(self.ln, self.sc[2 * i + 1], pos, e.text_seq_len, e.shift_w)
            ops.linear_fwd(self.ln, e.W(p + "w1"), self.h1, bias=e.P(p + "b1"), **e.mlp_act)
            self._branch_out(p, "m", self.h1, e.W(p + "w2"), e.P(p + "b2"), self.xmid, x_out)
            x_in, x_out = x_out, x_in
        e.final_ln(x_in, self.ln, self.mean, self.rstd, self.mf)
        e.vocab_gemm(self.ln, self.logit, bias=e.P("bout"))
        return self.logit

    # -------------------------------------------------------------------------------------------- CUDA-graph path
    def _step_dev(self, tokens, pos_dev=None):
        """self.step with the position (and the input token column) read on the device from pos_dev (default
        self.pos_dev, the image graphs' position)."""
        e = self.e
        pos_dev = self.pos_dev if pos_dev is None else pos_dev
        ops.embed_fwd_at_dev(tokens, e.embed_table(), e.pos_embedding(), self.x[0], pos_dev)
        x_in, x_out = self.x
        for i in range(e.L):
            p = f"l{i}."
            ops.layernorm_fwd(x_in, e.P(p + "ln1_g"), e.P(p + "ln1_b"), self.ln, self.mean, self.rstd, e.ln_eps)
            if e.shift_tokens:
                ops.shift_tokens_decode_dev(self.ln, self.sc[2 * i], pos_dev, e.text_seq_len, e.shift_w)
            if e.mlp[i]:
                self._branch_out(p, "a", self._gmlp_step(p, i, pos_dev=pos_dev), e.W(p + "gm_wout"),
                                 e.P(p + "gm_bout"), x_in, self.xmid)
            else:
                ops.linear_fwd(self.ln, e.W(p + "wqkv"), self.qkv)
                if e.rotary:
                    ops.rope_decode_dev(self.qkv, e.rope_table, pos_dev, e.H, e.dh, e.rotary_dim)
                if e.rotary_emb:
                    ops.rope_emb_decode_dev(self.qkv, e.rope_emb_table, pos_dev, e.H, e.dh)
                ops.attn_decode_dev(self.qkv, self.kc[i], self.vc[i], self.att, pos_dev, e.attn_scale,
                                    radius=e.radii[i], **e.axial_kw[i], **e.conv_kw[i], **e.block_sparse_kw[i])
                self._branch_out(p, "a", self.att, e.W(p + "wo"), e.P(p + "o_b"), x_in, self.xmid)
            ops.layernorm_fwd(self.xmid, e.P(p + "ln2_g"), e.P(p + "ln2_b"), self.ln, self.mean, self.rstd, e.ln_eps)
            if e.shift_tokens:
                ops.shift_tokens_decode_dev(self.ln, self.sc[2 * i + 1], pos_dev, e.text_seq_len, e.shift_w)
            ops.linear_fwd(self.ln, e.W(p + "w1"), self.h1, bias=e.P(p + "b1"), **e.mlp_act)
            self._branch_out(p, "m", self.h1, e.W(p + "w2"), e.P(p + "b2"), self.xmid, x_out)
            x_in, x_out = x_out, x_in
        e.final_ln(x_in, self.ln, self.mean, self.rstd, self.mf)
        e.vocab_gemm(self.ln, self.logit, bias=e.P("bout"))
        return self.logit

    def _filter(self, top_k, top_p, n_text=None):
        """(top_k, top_p) as the filtered kernel takes them, or None when neither truncates anything (the unfiltered
        kernels then run, exactly as without the arguments).  The draw is over the image_vocab_size image tokens, or
        with n_text over the n_text ids of the text window."""
        if top_k is not None and (isinstance(top_k, bool) or int(top_k) != top_k or top_k < 1):
            raise ValueError(f"top_k must be an integer >= 1 (or None), got {top_k!r}")
        if top_p is not None and not 0.0 < top_p <= 1.0:
            raise ValueError(f"top_p must lie in (0, 1] (or be None), got {top_p!r}")
        n = self.e.image_vocab_size if n_text is None else n_text
        k = 0 if top_k is None or top_k >= n else int(top_k)
        p = 1.0 if top_p is None else float(top_p)
        if k == 0 and p == 1.0:
            return None
        if n > FILTER_MAX_IDS:
            if n_text is None:
                raise ValueError(f"top_k / top_p filter at most {FILTER_MAX_IDS} image tokens, but image_vocab_size = "
                                 f"{n}; sample without a filter")
            raise ValueError(f"top_k / top_p filter at most {FILTER_MAX_IDS} ids, but the text window [0, "
                             f"image_offset) holds {n}; sample without a filter")
        return k, p

    @staticmethod
    def _guidance(scale):
        """The guidance scale as the guided kernel takes it, or None when guidance is off (None or 1.0: the plain
        sampler runs, exactly as without the argument)."""
        if scale is None:
            return None
        if isinstance(scale, bool) or not isinstance(scale, numbers.Real) or not math.isfinite(scale) or scale < 0:
            raise ValueError(f"guidance_scale must be a finite number >= 0 (or None), got {scale!r}")
        return None if float(scale) == 1.0 else float(scale)

    def _sample_guided(self, logits, u, tokens, inv_t, flt, gs, pos_dev=None):
        e = self.e
        lo, hi = e.image_offset, e.image_offset + e.image_vocab_size
        ops.sample_rows_guided(logits, u, tokens, lo, hi, inv_t, gs, *(flt or (0, 1.0)), pos_dev=pos_dev)

    def _capture(self, B, greedy, inv_t, flt, gs=None):
        """Two graphs over static buffers: the prompt step (teacher forcing: the next token is already in the token
        matrix) and the sampling step (step -> noise -> Gumbel-max into column pos + 1); both end by advancing pos_dev.
        B sampled rows; with guidance (gs) the steps run 2B rows (self._alloc(2 * B) first) and the noise has B."""
        e = self.e
        key = (B, greedy, inv_t, flt, gs)
        if getattr(self, "_graph_key", None) == key:
            return
        dev = e.device
        self.tokens = torch.zeros(2 * B if gs is not None else B, e.S, dtype=I32, device=dev)
        self.pos_dev = torch.zeros(1, dtype=I32, device=dev)
        lo, hi = e.image_offset, e.image_offset + e.image_vocab_size

        def sample(logits):
            if gs is not None:
                self._sample_guided(logits, self.u, self.tokens, inv_t, flt, gs, self.pos_dev)
            elif flt is None:
                ops.sample_rows_at(logits, self.u, self.tokens, lo, hi, inv_t, self.pos_dev)
            else:
                ops.sample_rows_filtered_at(logits, self.u, self.tokens, lo, hi, inv_t, *flt, self.pos_dev)

        self.u = None if greedy else torch.empty(B, hi - lo, dtype=F32, device=dev)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):     # eager warm-up: function attributes, tensor maps, lazy allocations
            logits = self._step_dev(self.tokens)
            if self.u is not None:
                self.u.uniform_(1e-9, 1.0)
            sample(logits)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.g_prompt, self.g_sample = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_prompt):
            self._step_dev(self.tokens)
            ops.incr_i32(self.pos_dev, 1)
        with torch.cuda.graph(self.g_sample):
            logits = self._step_dev(self.tokens)
            if self.u is not None:
                self.u.uniform_(1e-9, 1.0)          # default CUDA generator: graph-safe Philox offsets
            sample(logits)
            ops.incr_i32(self.pos_dev, 1)
        self._graph_key = key

    @torch.no_grad()
    def generate_graphed(self, text_ids, temperature=1.0, top_k=None, top_p=None, guidance_scale=None):
        """generate() with the per-position step replayed from CUDA graphs (position kept on the device): removes the
        ~45 us of Python / ctypes / launch overhead per kernel that bounds eager generation.  Noise comes from torch's
        default CUDA generator (seed it with torch.manual_seed).  Changing temperature, top_k, top_p or guidance_scale
        re-captures."""
        e = self.e
        B, TL = text_ids.shape
        assert TL == e.text_seq_len, f"expected {e.text_seq_len} text positions, got {TL}"
        flt = self._filter(top_k, top_p)
        gs = self._guidance(guidance_scale)
        self._alloc(2 * B if gs is not None else B)
        greedy = temperature is None or temperature <= 0
        inv_t = 1.0 if greedy else 1.0 / float(temperature)
        self._capture(B, greedy, inv_t, flt, gs)
        self.tokens.zero_()
        self.tokens[:B, :TL] = self._captions(text_ids)
        if gs is not None:
            self.tokens[B:, :TL] = self._uncond(B)
        self.pos_dev.zero_()
        for pos in range(e.S - 1):
            (self.g_prompt if pos + 1 < TL else self.g_sample).replay()
        return self.tokens[:B].clone()

    @torch.no_grad()
    def complete(self, text_ids, image_prefix=None, samples_per_prompt=1, temperature=1.0, top_k=None, top_p=None,
                 guidance_scale=None):
        """Image completion: text_ids int32 [B, text_seq_len] (device) and optionally image_prefix int32 [B, n], the
        first n (0 < n < image_seq_len) VAE codes in [0, image_vocab_size) in the VAE's row-major token order (e.g.
        vae.encode_tokens(img)[:, :n]).  Returns int32 [B * samples_per_prompt, text_seq_len + image_seq_len]: row
        b * samples_per_prompt + r is sample r of prompt b, the prompt (prefix offset by image_offset) followed by
        sampled image-token ids.

        The whole prompt (P = text_seq_len + n positions) runs once per distinct prompt as one batched forward pass
        (DalleEngine.prefill) that fills every replica's K/V cache; token P is drawn from its logits and the remaining
        positions replay the captured sampling step of generate_graphed.  temperature, top_k, top_p and guidance_scale
        mean what they mean for generate(); noise comes from torch's default CUDA generator (seed it with
        torch.manual_seed).  With guidance the one prefill runs 2B prompts, the captions and then as many padding
        captions, each followed by the same image prefix: its b * samples_per_prompt + r row order puts the conditional
        rows first and their unconditional twins second, the layout the guided sampler reads."""
        e = self.e
        if not torch.is_tensor(text_ids) or text_ids.dim() != 2 or text_ids.shape[1] != e.text_seq_len:
            raise ValueError(f"text_ids must be [B, {e.text_seq_len}], got "
                             f"{tuple(text_ids.shape) if torch.is_tensor(text_ids) else type(text_ids).__name__}")
        B, TL = text_ids.shape
        rep = samples_per_prompt
        if isinstance(rep, bool) or int(rep) != rep or rep < 1:
            raise ValueError(f"samples_per_prompt must be an integer >= 1, got {rep!r}")
        rep = int(rep)
        n = 0
        if image_prefix is not None:
            if not torch.is_tensor(image_prefix) or image_prefix.dim() != 2 or image_prefix.shape[0] != B:
                raise ValueError(f"image_prefix must be [{B}, n]")
            n = image_prefix.shape[1]
            if not 0 < n < e.image_seq_len:
                raise ValueError(f"image_prefix length {n} outside (0, {e.image_seq_len})")
            if int(image_prefix.min()) < 0 or int(image_prefix.max()) >= e.image_vocab_size:
                raise ValueError(f"image_prefix codes must lie in [0, {e.image_vocab_size})")
        flt = self._filter(top_k, top_p)
        gs = self._guidance(guidance_scale)
        P, R = TL + n, B * rep
        self._alloc(2 * R if gs is not None else R)
        greedy = temperature is None or temperature <= 0
        inv_t = 1.0 if greedy else 1.0 / float(temperature)
        # capture before the prefill (the capture's warm-up step writes the caches), and without moving the default
        # generator (its warm-up draws noise): a seeded call then samples the same whether or not it had to capture
        rng = torch.cuda.get_rng_state(e.device)
        self._capture(R, greedy, inv_t, flt, gs)
        torch.cuda.set_rng_state(rng, e.device)
        prompt = torch.empty(2 * B if gs is not None else B, P, dtype=I32, device=e.device)
        prompt[:B, :TL] = self._captions(text_ids)
        if gs is not None:
            prompt[B:, :TL] = self._uncond(B)
        if n:   # (with guidance the padding-caption prompts continue with the same image prefix)
            prompt[:, TL:] = (image_prefix.to(device=e.device, dtype=I32) + e.image_offset).repeat(len(prompt) // B, 1)
        logits = e.prefill(prompt, self.kc, self.vc, rep, shift_caches=self.sc)
        lo, hi = e.image_offset, e.image_offset + e.image_vocab_size
        if self.u is not None:
            self.u.uniform_(1e-9, 1.0)
        if gs is not None:
            self._sample_guided(logits, self.u, self.tok.view(-1, 1), inv_t, flt, gs)
        elif flt is None:
            ops.sample_rows(logits, self.u, self.tok, lo, hi, inv_t)
        else:
            ops.sample_rows_filtered(logits, self.u, self.tok, lo, hi, inv_t, *flt)
        self.tokens.zero_()
        self.tokens[:, :P] = prompt.repeat_interleave(rep, 0)
        self.tokens[:, P] = self.tok
        self.pos_dev.fill_(P)
        for _ in range(P, e.S - 1):
            self.g_sample.replay()
        return self.tokens[:R].clone()

    # ------------------------------------------------------------------------------------------- caption generation
    def caption_lengths(self, text_ids):
        """Prefix lengths n_b of caption rows text_ids int [B, text_seq_len]: the ids before the first padding_id
        (text_seq_len when there is none), as an int32 tensor on text_ids' device.  Raises ValueError for a wrong shape,
        an id outside [0, text_vocab_size) or an empty prefix."""
        e = self.e
        if not torch.is_tensor(text_ids) or text_ids.dim() != 2 or text_ids.shape[1] != e.text_seq_len or \
                text_ids.shape[0] < 1 or text_ids.dtype.is_floating_point or text_ids.dtype == torch.bool:
            raise ValueError(f"text_ids must be an integer tensor [B >= 1, {e.text_seq_len}], got "
                             f"{tuple(text_ids.shape) if torch.is_tensor(text_ids) else type(text_ids).__name__}")
        if int(text_ids.min()) < 0 or int(text_ids.max()) >= e.text_vocab_size:
            raise ValueError(f"caption ids must lie in [0, {e.text_vocab_size})")
        pad = text_ids == self.padding_id
        lens = torch.where(pad.any(1), pad.to(I32).argmax(1), e.text_seq_len).to(I32)
        empty = (lens == 0).nonzero().flatten().tolist()
        if empty:
            raise ValueError(f"caption rows {empty} start with padding_id {self.padding_id}: an empty prefix has "
                             "nothing to continue from (position 0 is never a training target; DALLE-pytorch starts "
                             "such a caption from id 0)")
        return lens

    def _capture_text(self, B, greedy, inv_t, flt):
        """The text step graph over its own static buffers (token matrix, prompt, prompt lengths, position, noise):
        step -> noise -> draw over the text window into column pos + 1 -> caption_next_at -> advance the position."""
        e = self.e
        key = (B, greedy, inv_t, flt)
        if self._text_key == key:
            return
        dev, TL, hi = e.device, e.text_seq_len, e.image_offset
        self.t_tokens = torch.zeros(B, TL, dtype=I32, device=dev)
        self.t_prefix = torch.zeros(B, TL, dtype=I32, device=dev)
        self.t_lens = torch.full((B,), TL, dtype=I32, device=dev)
        self.t_pos = torch.zeros(1, dtype=I32, device=dev)
        self.t_u = None if greedy else torch.empty(B, hi, dtype=F32, device=dev)

        def step():
            logits = self._step_dev(self.t_tokens, self.t_pos)
            if self.t_u is not None:
                self.t_u.uniform_(1e-9, 1.0)        # default CUDA generator: graph-safe Philox offsets
            if flt is None:
                ops.sample_rows_at(logits, self.t_u, self.t_tokens, 0, hi, inv_t, self.t_pos)
            else:
                ops.sample_rows_filtered_at(logits, self.t_u, self.t_tokens, 0, hi, inv_t, *flt, self.t_pos)
            ops.caption_next_at(self.t_tokens, self.t_prefix, self.t_lens, self.t_pos, TL, e.text_vocab_size,
                                self.padding_id, e.pad_base)

        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):     # eager warm-up, as in _capture
            step()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.g_text = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_text):
            step()
            ops.incr_i32(self.t_pos, 1)
        self._text_key = key

    @torch.no_grad()
    def generate_texts(self, text_ids, temperature=1.0, top_k=None, top_p=None):
        """Caption completion (DALLE-pytorch's generate_texts): text_ids int [B, text_seq_len], captions padded with
        padding_id as generate_dalle.pad_captions pads them -> int32 [B, text_seq_len] (device) in the same form,
        ready for generate, generate_graphed or complete.

        Row b's prefix is its ids before the first padding_id; its length n_b must be >= 1 (an empty prefix raises
        ValueError: position 0 is never a training target, so there is nothing to draw it from; DALLE-pytorch starts
        from id 0).  Ids outside [0, text_vocab_size) raise ValueError.  Columns c < n_b come back bit for bit.  Column
        c >= n_b is drawn from the model's logits at position c - 1 restricted to the text window [0, image_offset)
        (text_vocab_size ids, plus the text_seq_len per-position pads with per_position_padding): the logits mask's
        text window, whether the model was trained with logits_mask or not.  The draw applies temperature, then top_k,
        then top_p, then the Gumbel-max: the image sampler's semantics and kernels; temperature 0 or None is greedy.
        A drawn padding token (padding_id, or with per-position padding any id >= text_vocab_size) ends the caption:
        that column and every later one are padding_id in the result (in the decoder's token matrix, each column's
        per-position pad), as training data is right-padded.  Rows with n_b = text_seq_len come back unchanged.

        One prefill runs the common prefix P = min_b n_b, column P is drawn from its logits, and the captured text step
        continues to the last text column; rows with a longer prefix are teacher-forced up to it.  Noise comes from
        torch's default CUDA generator (seed it with torch.manual_seed); a seeded call draws the same whether or not it
        had to capture.  There is no guidance and no samples_per_prompt: repeat the prompt rows for several samples."""
        e = self.e
        lens = self.caption_lengths(text_ids)
        flt = self._filter(top_k, top_p, n_text=e.image_offset)
        B, TL = text_ids.shape
        text_ids = text_ids.to(device=e.device, dtype=I32).contiguous()
        P = int(lens.min())
        if P == TL:
            return text_ids.clone()
        greedy = temperature is None or temperature <= 0
        inv_t = 1.0 if greedy else 1.0 / float(temperature)
        self._alloc(B)
        rng = torch.cuda.get_rng_state(e.device)   # as in complete: the capture's warm-up draws noise
        self._capture_text(B, greedy, inv_t, flt)
        torch.cuda.set_rng_state(rng, e.device)
        prompt = self._captions(text_ids)
        self.t_prefix.copy_(prompt)
        self.t_lens.copy_(lens)
        logits = e.prefill(prompt[:, :P].contiguous(), self.kc, self.vc, 1, shift_caches=self.sc)
        if self.t_u is not None:
            self.t_u.uniform_(1e-9, 1.0)
        if flt is None:
            ops.sample_rows(logits, self.t_u, self.tok, 0, e.image_offset, inv_t)
        else:
            ops.sample_rows_filtered(logits, self.t_u, self.tok, 0, e.image_offset, inv_t, *flt)
        self.t_tokens.copy_(prompt)
        self.t_tokens[:, P] = self.tok
        ops.caption_next(self.t_tokens, self.t_prefix, self.t_lens, P - 1, TL, e.text_vocab_size, self.padding_id,
                         e.pad_base)
        self.t_pos.fill_(P)
        for _ in range(P, TL - 1):
            self.g_text.replay()
        out = self.t_tokens.clone()
        return out.masked_fill_(out >= e.text_vocab_size, self.padding_id) if e.per_position_padding else out

    @torch.no_grad()
    def generate(self, text_ids, temperature=1.0, generator=None, return_logits=False, top_k=None, top_p=None,
                 guidance_scale=None):
        """text_ids int32 [B, text_seq_len] (device) -> int32 [B, text_seq_len + image_seq_len]: the prompt followed by
        image_seq_len sampled image-token ids (already offset by the engine's image_offset, as in training).

        top_k (>= 1) keeps the k most likely image tokens (all of a tie at the k-th), top_p (in (0, 1]) the smallest
        set of them whose probability mass after temperature reaches p (nucleus sampling); with both, top-k applies
        first.  None disables either; no filter at all runs the unfiltered sampler.

        guidance_scale s (finite, >= 0; None or 1 = off): classifier-free guidance, each image token drawn from
        u + s (c - u) of the logits given the caption (c) and given a padding-only caption (u).  With guidance,
        return_logits returns all 2B rows of each step, the conditional rows first."""
        e = self.e
        B, TL = text_ids.shape
        assert TL == e.text_seq_len, f"expected {e.text_seq_len} text positions, got {TL}"
        flt = self._filter(top_k, top_p)
        gs = self._guidance(guidance_scale)
        rows = 2 * B if gs is not None else B
        self._alloc(rows)
        out = torch.empty(rows, e.S, dtype=I32, device=e.device)
        out[:B, :TL] = self._captions(text_ids)
        if gs is not None:
            out[B:, :TL] = self._uncond(B)
        lo, hi = e.image_offset, e.image_offset + e.image_vocab_size
        greedy = temperature is None or temperature <= 0
        inv_t = 1.0 if greedy else 1.0 / float(temperature)
        kept = [] if return_logits else None
        for pos in range(e.S - 1):
            cur = out[:, pos].contiguous()
            logits = self.step(cur, pos)
            if return_logits:
                kept.append(logits[:, :e.V].clone())
            if pos + 1 < TL:
                continue  # next position is part of the prompt: teacher forcing
            u = None
            if not greedy:
                u = torch.empty(B, hi - lo, dtype=F32, device=e.device).uniform_(1e-9, 1.0, generator=generator)
            if gs is not None:
                self._sample_guided(logits, u, self.tok.view(-1, 1), inv_t, flt, gs)
            elif flt is None:
                ops.sample_rows(logits, u, self.tok, lo, hi, inv_t)
            else:
                ops.sample_rows_filtered(logits, u, self.tok, lo, hi, inv_t, *flt)
            out[:, pos + 1] = self.tok
        out = out[:B] if gs is not None else out
        return (out, kept) if return_logits else out
