"""Model classes with the reference's constructor / forward signatures (src/dalle_mtf/models.py:141-416 DALLE,
src/vae_tf/models.py:46-184 DiscreteVAE), backed by the engines.  These are the objects a user of the reference
instantiates directly; training goes through model_fns.* which drive the same engines.
"""
import torch

from . import lib as L
from .dalle_engine import DalleEngine
from .model_fns import activation_function, attention_layers, block_sparse_options, conv_kernel, dropout_rates, \
    gated_mlp, input_embedding, layer_scale, logits_mask, loss_weights, rotary_emb, rotary_embedding, sandwich_norm, \
    share_input_output_emb, shared_attn_ids, shared_ff_ids, shift_tokens, stable, validate_kl_weight
from .model_fns import build_vae_engine, vae_architecture
from .utils import fetch_model_params, latest_checkpoint, load_checkpoint, local_path
from .model_fns import reconstruction_loss as _reconstruction_loss


class DALLE:
    def __init__(self, n_embd, text_vocab_size=12800, image_vocab_size=512, text_seq_len=256, image_seq_len=1024,
                 n_layers=6, n_heads=8, batch_size=32, bf_16=True, attn_mask=None, mode="train",
                 is_incremental_inference=False, context=None, loss_fn=None, params=None, eos_token_id=None,
                 activation_fn=None):
        if attn_mask is not None or loss_fn is not None or activation_fn is not None:
            raise L.DB200Error("custom attn_mask / loss_fn / activation_fn are not supported: the fused kernels "
                               "implement the reference defaults (causal mask, softmax CE, ReLU); select GELU with "
                               "params[\"activation_function\"] = \"gelu\"")
        if is_incremental_inference or context is not None:
            raise NotImplementedError("incremental inference is stubbed in the reference too (src/model_fns.py:135)")
        params = params or {}
        attention_types, local_radius = attention_layers({**params, "n_layers": n_layers})
        conv_k = conv_kernel(params)
        sparse = block_sparse_options(params)
        weights, z_loss = loss_weights(params)
        pos_scheme, per_pos, _ = input_embedding({**params, "text_vocab_size": text_vocab_size})
        activation = activation_function(params)
        gated = gated_mlp(params)
        shift = shift_tokens(params, image_seq_len)
        sandwich = sandwich_norm(params)
        scale = layer_scale(params)
        stab = stable(params)
        tied = share_input_output_emb(params)
        attn_ids, ff_ids = shared_attn_ids(params), shared_ff_ids(params)
        mask = logits_mask(params)
        rotary_dim, rotary_base = rotary_embedding(params, n_embd, n_heads)
        rot_emb = rotary_emb(params, image_seq_len)
        self.n_embd, self.n_layers, self.n_heads = n_embd, n_layers, n_heads
        self.text_vocab_size, self.image_vocab_size = text_vocab_size, image_vocab_size
        self.text_seq_len, self.image_seq_len = text_seq_len, image_seq_len
        self.total_seq_dim = text_seq_len + image_seq_len
        # per-position padding: text_seq_len padding tokens follow the text vocabulary
        self.total_tokens = text_vocab_size + (text_seq_len if per_pos else 0) + image_vocab_size + 1
        self.eos_token_id = self.total_tokens - 1 if eos_token_id is None else eos_token_id
        self.batch_size, self.bf_16, self.mode = batch_size, bf_16, mode
        self.engine = DalleEngine(n_embd, n_layers, n_heads, text_vocab_size, image_vocab_size, text_seq_len,
                                  image_seq_len, recompute_grad=bool(params.get("recompute_grad")) and mode == "train",
                                  dropout=dropout_rates(params), dropout_seed=params.get("seed") or 0,
                                  attention_types=attention_types, local_attention_radius=local_radius,
                                  conv_attention_kernel=conv_k, loss_weights=weights, z_loss=z_loss,
                                  image_position_embedding=None if rot_emb else pos_scheme,
                                  per_position_padding=per_pos, activation=activation, logits_mask=mask,
                                  rotary_dim=rotary_dim, rotary_base=rotary_base, gated_mlp=gated, shift_tokens=shift,
                                  sandwich_norm=sandwich, layer_scale=scale, stable=stab,
                                  share_input_output_emb=tied, shared_attn_ids=attn_ids, shared_ff_ids=ff_ids,
                                  rotary_emb=rot_emb, **sparse)
        self.loss_parts = None   # weighted loss: device [3] of the last forward (text / image mean CE, mean z-term)
        self._step = 0   # mode "train": each forward draws the dropout masks of the next step
        self.engine.eos_token_id = self.eos_token_id
        self.engine.init_params(seed=params.get("seed") or 0)
        self.padding_id = params.get("padding_id")   # caption of guided sampling's unconditional rows (None: tv - 1)

    def forward(self, features, return_loss=True, return_logits=False):
        """features = {"tokens": int [B, S]}.  Returns what the reference returns (models.py:397-416):
        logits | (loss, loss_batch) | (loss, loss_batch, logits), as device tensors (loss fp32 scalar).
        With params text_loss_weight / image_loss_weight / z_loss, loss is the weighted loss over this batch,
        loss_batch holds CE + z_loss * lse^2 per position, and self.loss_parts the text-row mean CE, the image-row mean
        CE and the mean z-term."""
        tokens = features["tokens"] if isinstance(features, dict) else features
        tokens = tokens.to(device=self.engine.device, dtype=torch.int32).contiguous()
        B, S = tokens.shape
        if not return_loss:
            return self.engine.logits(tokens)
        e = self.engine
        acc = torch.zeros(4 if e.weighted_loss else 1, dtype=torch.float32, device=e.device)
        step = None
        if self.mode == "train":   # dropout only in train mode (models.py:198, 215, 290, 312, 318)
            step, self._step = self._step, self._step + 1
        e.forward(tokens, loss_accum=acc, step=step)
        if e.weighted_loss:         # slot 0 is the loss itself (coefficients of a batch of B sequences)
            loss = acc[:1]
            self.loss_parts = acc[1:4] * torch.tensor(e.loss_part_scales(B), dtype=torch.float32, device=e.device)
        else:
            loss = acc / float(B * S)   # reduce_mean over every position (models.py:353-354); scalar glue only
        loss_batch = self.engine._bufs["loss_rows"].view(B, S)
        if return_logits:
            return loss, loss_batch, self.engine.logits(tokens)
        return loss, loss_batch


    def _get_sampler(self):
        from .sampling import DalleSampler
        if getattr(self, "_sampler", None) is None:
            self._sampler = DalleSampler(self.engine, padding_id=self.padding_id)
        return self._sampler

    def sample(self, text_ids, temperature=1.0, generator=None, top_k=None, top_p=None, guidance_scale=None):
        """Autoregressive generation with a K/V cache ("next" row N4; the reference stubs inference):
        text_ids int [B, text_seq_len] -> int32 [B, text_seq_len + image_seq_len], image positions sampled from
        softmax(logits / temperature) restricted to the image-token ids (temperature 0 = greedy), optionally truncated
        to its top_k ids and / or its top_p nucleus, optionally with classifier-free guidance of scale guidance_scale
        against a padding-only caption (params["padding_id"], default text_vocab_size - 1) (DalleSampler.generate)."""
        text_ids = text_ids.to(device=self.engine.device, dtype=torch.int32).contiguous()
        return self._get_sampler().generate(text_ids, temperature, generator, top_k=top_k, top_p=top_p,
                                            guidance_scale=guidance_scale)

    def complete(self, text_ids, image_prefix=None, samples_per_prompt=1, temperature=1.0, top_k=None, top_p=None,
                 guidance_scale=None):
        """Image completion (DalleSampler.complete): text_ids int [B, text_seq_len] plus optionally the first n VAE codes
        of each image, image_prefix int [B, n] -> int32 [B * samples_per_prompt, text_seq_len + image_seq_len].  The
        prompt is prefilled in one forward pass; noise comes from torch's default CUDA generator."""
        text_ids = text_ids.to(device=self.engine.device, dtype=torch.int32).contiguous()
        if image_prefix is not None:
            image_prefix = image_prefix.to(device=self.engine.device, dtype=torch.int32).contiguous()
        return self._get_sampler().complete(text_ids, image_prefix, samples_per_prompt, temperature, top_k, top_p,
                                            guidance_scale)

    def generate_texts(self, text_ids, temperature=1.0, top_k=None, top_p=None):
        """Caption completion (DalleSampler.generate_texts, DALLE-pytorch's generate_texts): text_ids int [B,
        text_seq_len], each row a non-empty prefix padded with padding_id -> int32 [B, text_seq_len], the prefix kept
        and the rest drawn from the text window until a padding token ends the caption (temperature 0 = greedy)."""
        return self._get_sampler().generate_texts(text_ids, temperature, top_k, top_p)


class DiscreteVAE:
    def __init__(self, num_tokens, dimensions, convblocks=None, dim=512, hidden_dim=64, input_channels=3,
                 recompute_grad=False, use_bf16=False, stack_factor=1, kl_loss_weight=None, reconstruction_loss=None,
                 architecture=None, n_hid=None, n_blk_per_group=None, group_count=None, n_init=None):
        """kl_loss_weight (extension; None: the reference's objective): beta of the KL term, a finite real >= 0.  With
        it, forward(..., return_recon_loss=True) returns MSE + beta * KL, KL the mean over the batch's latent rows of
        KL(softmax(logits) || Uniform(K)), and leaves the device [2] (MSE, KL) in self.loss_parts.

        reconstruction_loss (extension; None or "mse": the reference's MSE): "logit_laplace" makes the reconstruction
        term the mean logit-Laplace NLL; forward then returns the image-space output and, with return_recon_loss, the
        objective NLL (+ beta * KL), leaving the device (NLL, image-space MSE) or (NLL, image-space MSE, KL) in
        self.loss_parts.

        architecture (extension; None or "reference": the reference's network, sized by convblocks): "dalle_paper"
        builds the DALL-E paper's network instead, sized by n_hid, n_blk_per_group, group_count and n_init (None:
        256, 2, 4, 128); convblocks must then be None and stack_factor 1 (model_fns.vae_architecture)."""
        self.kl_loss_weight, _ = validate_kl_weight(kl_loss_weight)
        cfg = {"architecture": architecture, "convblocks": convblocks, "stack_factor": stack_factor,
               "n_hid": n_hid, "n_blk_per_group": n_blk_per_group, "group_count": group_count, "n_init": n_init,
               "num_tokens": num_tokens, "input_channels": input_channels, "use_bf16": use_bf16,
               "recompute_grad": recompute_grad, "reconstruction_loss": reconstruction_loss}
        if vae_architecture(cfg, dimensions) is None and convblocks is None:
            raise ValueError("DiscreteVAE: the reference network needs convblocks")
        self.reconstruction_loss = _reconstruction_loss(reconstruction_loss)
        self.loss_parts = None
        self.num_tokens, self.dim, self.hdim = num_tokens, dim, hidden_dim   # dim / hidden_dim have no effect (ref too)
        self.H = self.W = dimensions
        self.convblocks = convblocks
        self.num_ch = input_channels
        self.stack_factor = stack_factor
        self.engine = build_vae_engine(cfg, dimensions, "cuda", kl=self.kl_loss_weight is not None)
        self.engine.init_params(0)
        self._gen = torch.Generator(device=self.engine.device).manual_seed(1234)

    def forward(self, features, return_recon_loss=False, return_logits=False, hard_gumbel=True, temperature=1.):
        img = features["inputs"] if isinstance(features, dict) else features
        img = img.to(device=self.engine.device, dtype=torch.float32).contiguous()
        e = self.engine
        if return_logits:
            B = img.shape[0]
            return e.encode_logits(img).view(B, e.hw, e.hw, e.K)
        rows = img.shape[0] * e.hw * e.hw
        u = torch.empty(rows, e.K, dtype=torch.float32, device=e.device).uniform_(1e-9, 1.0, generator=self._gen)
        kl = self.kl_loss_weight is not None
        ll = e.logit_laplace
        acc = torch.zeros(3 if ll else (2 if kl else 1), dtype=torch.float32, device=e.device)  # [recon, KL, MSE]
        out = e.forward(img, u, temperature, hard_gumbel, loss_accum=acc[:1], kl_weight=self.kl_loss_weight,
                        kl_accum=acc[1:2] if kl else None, mse_accum=acc[2:3] if ll else None)
        if not return_recon_loss:
            return out
        if ll:
            self.loss_parts = torch.cat([acc[:1], acc[2:3]] + ([acc[1:2]] if kl else []))
            return (acc[:1] + self.kl_loss_weight * acc[1:2] if kl else acc[:1]), out
        if kl:                     # scalar glue: the objective from the two device sums
            self.loss_parts = acc
            return acc[:1] + self.kl_loss_weight * acc[1:], out
        return acc, out

    def decode(self, image_token_ids, offset=0):
        """Sampled image-token ids [B, image_seq_len] (minus `offset`, e.g. DALLE's text_vocab_size) -> images fp32 NHWC:
        one-hot codes through the tied codebook and the decoder (src/vae_tf/models.py:123-163)."""
        ids = image_token_ids.to(device=self.engine.device, dtype=torch.int32).contiguous()
        return self.engine.decode_tokens(ids, offset)


class VQGanVAE:
    def __init__(self, vae_model, checkpoint=None):
        """DALLE-pytorch's VQGanVAE over a taming VQGAN imported with tools/import_vqgan.py.  vae_model is a VAE config
        name or path with architecture "vqgan" (e.g. "vae_vqgan_f16_16384_b200"); checkpoint is this project's
        checkpoint file (default: the latest one under the config's model_path).

        Images follow this project's convention, f32 NHWC in [-1, 1], not DALLE-pytorch's NCHW in [0, 1]:
        get_codebook_indices takes such images and decode returns them."""
        params = fetch_model_params(vae_model) if isinstance(vae_model, str) else vae_model
        if params.get("architecture") != "vqgan":
            raise ValueError(f"VQGanVAE: architecture = {params.get('architecture')!r}, expected \"vqgan\"")
        ckpt = checkpoint or (latest_checkpoint(params["model_path"]) if params.get("model_path") else None)
        if ckpt is None:
            raise ValueError(f"VQGanVAE: no checkpoint under {params.get('model_path')!r}: import one with "
                             "tools/import_vqgan.py")
        self.engine = build_vae_engine(params, params["dataset"]["image_size"], "cuda")
        state = load_checkpoint(local_path(ckpt))
        self.engine.load_params({k[len("vae/"):]: v for k, v in state.items() if k.startswith("vae/")})
        e = self.engine
        self.num_tokens, self.image_size = e.K, e.img_H
        self.num_layers = len(params["ch_mult"]) - 1      # DALLE-pytorch: log2(image_size / grid side)
        self.channels = 3

    def get_codebook_indices(self, img):
        """img f32 NHWC [B, H, W, 3] in [-1, 1] -> int32 [B, h * w] nearest codes (raster order)."""
        img = img.to(device=self.engine.device, dtype=torch.float32).contiguous()
        return self.engine.encode_tokens(img).clone()

    def decode(self, img_seq, offset=0):
        """Codes [B, h * w] (minus `offset`) -> images f32 NHWC [B, H, W, 3] in [-1, 1]."""
        ids = img_seq.to(device=self.engine.device, dtype=torch.int32).contiguous()
        return self.engine.decode_tokens(ids, offset).clone()
