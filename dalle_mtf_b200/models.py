"""Model classes with the reference's constructor / forward signatures (src/dalle_mtf/models.py:141-416 DALLE,
src/vae_tf/models.py:46-184 DiscreteVAE), backed by the engines.  These are the objects a user of the reference
instantiates directly; training goes through model_fns.* which drive the same engines.
"""
import torch

from . import lib as L
from .dalle_engine import DalleEngine
from .vae_engine import VaeEngine


class DALLE:
    def __init__(self, n_embd, text_vocab_size=12800, image_vocab_size=512, text_seq_len=256, image_seq_len=1024,
                 n_layers=6, n_heads=8, batch_size=32, bf_16=True, attn_mask=None, mode="train",
                 is_incremental_inference=False, context=None, loss_fn=None, params=None, eos_token_id=None,
                 activation_fn=None):
        if attn_mask is not None or loss_fn is not None or activation_fn is not None:
            raise L.DB200Error("custom attn_mask / loss_fn / activation_fn are not supported: the fused kernels "
                               "implement the reference defaults (causal mask, softmax CE, ReLU)")
        if is_incremental_inference or context is not None:
            raise NotImplementedError("incremental inference is stubbed in the reference too (src/model_fns.py:135)")
        params = params or {}
        self.n_embd, self.n_layers, self.n_heads = n_embd, n_layers, n_heads
        self.text_vocab_size, self.image_vocab_size = text_vocab_size, image_vocab_size
        self.text_seq_len, self.image_seq_len = text_seq_len, image_seq_len
        self.total_seq_dim = text_seq_len + image_seq_len
        self.total_tokens = text_vocab_size + image_vocab_size + 1
        self.eos_token_id = self.total_tokens - 1 if eos_token_id is None else eos_token_id
        self.batch_size, self.bf_16, self.mode = batch_size, bf_16, mode
        for k in ("embed_dropout", "attention_dropout", "residual_dropout"):
            if params.get(k):
                raise L.DB200Error(f"{k} > 0 is not implemented (every reference config leaves it at 0)")
        self.engine = DalleEngine(n_embd, n_layers, n_heads, text_vocab_size, image_vocab_size, text_seq_len,
                                  image_seq_len, recompute_grad=bool(params.get("recompute_grad")) and mode == "train")
        self.engine.eos_token_id = self.eos_token_id
        self.engine.init_params(seed=params.get("seed") or 0)

    def forward(self, features, return_loss=True, return_logits=False):
        """features = {"tokens": int [B, S]}.  Returns what the reference returns (models.py:397-416):
        logits | (loss, loss_batch) | (loss, loss_batch, logits), as device tensors (loss fp32 scalar)."""
        tokens = features["tokens"] if isinstance(features, dict) else features
        tokens = tokens.to(device=self.engine.device, dtype=torch.int32).contiguous()
        B, S = tokens.shape
        if not return_loss:
            return self.engine.logits(tokens)
        acc = torch.zeros(1, dtype=torch.float32, device=self.engine.device)
        self.engine.forward(tokens, loss_accum=acc)
        loss = acc / float(B * S)   # reduce_mean over every position (models.py:353-354); scalar glue only
        loss_batch = self.engine._bufs["loss_rows"].view(B, S)
        if return_logits:
            return loss, loss_batch, self.engine.logits(tokens)
        return loss, loss_batch


    def sample(self, text_ids, temperature=1.0, generator=None):
        """Autoregressive generation with a K/V cache ("next" row N4; the reference stubs inference):
        text_ids int [B, text_seq_len] -> int32 [B, text_seq_len + image_seq_len], image positions sampled from
        softmax(logits / temperature) restricted to the image-token ids (temperature 0 = greedy)."""
        from .sampling import DalleSampler
        if getattr(self, "_sampler", None) is None:
            self._sampler = DalleSampler(self.engine)
        text_ids = text_ids.to(device=self.engine.device, dtype=torch.int32).contiguous()
        return self._sampler.generate(text_ids, temperature, generator)


class DiscreteVAE:
    def __init__(self, num_tokens, dimensions, convblocks, dim=512, hidden_dim=64, input_channels=3,
                 recompute_grad=False, use_bf16=False, stack_factor=1):
        self.num_tokens, self.dim, self.hdim = num_tokens, dim, hidden_dim   # dim / hidden_dim have no effect (ref too)
        self.H = self.W = dimensions
        self.convblocks = convblocks
        self.num_ch = input_channels
        self.stack_factor = stack_factor
        self.engine = VaeEngine(num_tokens, dimensions, convblocks, input_channels, use_bf16, recompute_grad,
                                stack_factor)
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
        acc = torch.zeros(1, dtype=torch.float32, device=e.device)
        out = e.forward(img, u, temperature, hard_gumbel, loss_accum=acc)
        if not return_recon_loss:
            return out
        return acc, out

    def decode(self, image_token_ids, offset=0):
        """Sampled image-token ids [B, image_seq_len] (minus `offset`, e.g. DALLE's text_vocab_size) -> images fp32 NHWC:
        one-hot codes through the tied codebook and the decoder (src/vae_tf/models.py:123-163)."""
        ids = image_token_ids.to(device=self.engine.device, dtype=torch.int32).contiguous()
        return self.engine.decode_tokens(ids, offset)
