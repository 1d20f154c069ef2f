"""ctypes binding of libdalle_b200.so (the C ABI declared in include/dalle_b200.h).

The library is built in-tree by ``dalle_mtf_b200.build.build()`` (nvcc, sm_90a only).  There is no CPU fallback
and no PyTorch-eager fallback: if the shared object is missing, or the device is not an H100 (sm_90), every op
raises.  PyTorch is used only for device memory, streams and torch.distributed.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# DB200_LIB: load another build of the library (development: `make DEV=1 LIB=../libdalle_b200_dev.so`)
LIB_PATH = os.environ.get("DB200_LIB") or os.path.join(_HERE, "libdalle_b200.so")

c_int = ctypes.c_int
c_i64 = ctypes.c_int64
c_f32 = ctypes.c_float
c_vp = ctypes.c_void_p
c_sz = ctypes.c_size_t
c_u64 = ctypes.c_uint64

EPI_STORE, EPI_ATOMIC, EPI_RELU_BWD, EPI_CE_STATS, EPI_CE_GRAD = 0, 1, 2, 3, 4
ACT_RELU, ACT_GELU = 0, 1            # the gated MLP's gate nonlinearity (db200_gemm_bf16_glu*)


class GemmEpilogue(ctypes.Structure):
    """Mirror of ``struct db200_gemm_epilogue``."""
    _fields_ = [
        ("mode", ctypes.c_int32), ("out_f32", ctypes.c_int32), ("relu", ctypes.c_int32), ("split_k", ctypes.c_int32),
        ("alpha", c_f32),
        ("bias", c_vp), ("residual", c_vp), ("ldr", c_i64), ("aux", c_vp), ("ldaux", c_i64),
        ("labels", c_vp), ("part_max", c_vp), ("part_sum", c_vp), ("label_logit", c_vp), ("lse", c_vp),
        ("n_valid", ctypes.c_int32), ("reserved", ctypes.c_int32), ("colsum", c_vp),
        ("workspace", c_vp), ("workspace_bytes", c_i64),
    ]


class Dropout(ctypes.Structure):
    """Mirror of ``struct db200_dropout`` (one dropout site of one step; see include/dalle_b200.h, D0)."""
    _fields_ = [("seed", c_u64), ("step", ctypes.c_uint32), ("site", ctypes.c_uint32), ("threshold", ctypes.c_uint32),
                ("scale", c_f32), ("row0", c_i64)]


DROPOUT_ELEMENTWISE, DROPOUT_ATTENTION = 0, 1
SITE_WTE, SITE_WPE = 0, 1
SITE_CAPTION = 0xFFFFFFFF   # caption dropout (db200_assemble_tokens_ex): one decision per sequence


def dropout_site_attn(layer):
    return 2 + 3 * layer


def dropout_site_attn_out(layer):
    return 3 + 3 * layer


def dropout_site_mlp_out(layer):
    return 4 + 3 * layer


def dropout_threshold(rate):
    """Keep iff word >= floor(rate * 2^32) (computed in double); kept values are scaled by float(1 / (1 - rate))."""
    rate = float(rate)
    if not 0.0 <= rate < 1.0:
        raise ValueError(f"dropout rate {rate} outside [0, 1)")
    return int(rate * 4294967296.0), float(1.0 / (1.0 - rate))


def make_dropout(rate, seed, step, site, row0):
    """db200_dropout for one site, or None when rate == 0 (the kernels without dropout run)."""
    thr, scale = dropout_threshold(rate)
    if thr == 0:
        return None
    d = Dropout()
    d.seed, d.step, d.site, d.threshold, d.scale, d.row0 = int(seed) & (2 ** 64 - 1), int(step), int(site), thr, \
        scale, int(row0)
    return d


class CeWeights(ctypes.Structure):
    """Mirror of ``struct db200_ce_weights`` (weighted cross-entropy: per-row class coefficients and the z-loss)."""
    _fields_ = [("period", ctypes.c_int32), ("text_rows", ctypes.c_int32), ("a_text", c_f32), ("a_image", c_f32),
                ("z_loss", c_f32)]


def make_ce_weights(period, text_rows, a_text, a_image, z_loss):
    w = CeWeights()
    w.period, w.text_rows, w.a_text, w.a_image, w.z_loss = int(period), int(text_rows), float(a_text), \
        float(a_image), float(z_loss)
    return w


class ConvDesc(ctypes.Structure):
    """Mirror of ``struct db200_conv_desc``."""
    _fields_ = [(n, ctypes.c_int32) for n in
                ("N", "H", "W", "Cin", "Ho", "Wo", "Cout", "KH", "KW", "stride", "transposed", "act_f32", "relu",
                 "reserved")]


# name -> argtypes (restype is always int unless listed in _RESTYPES)
_SIGNATURES = {
    "db200_version": [],
    "db200_device_check": [],
    "db200_embed_fwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int],
    "db200_embed_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_i64],
    "db200_embed_fwd_ex": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, ctypes.POINTER(Dropout),
                           ctypes.POINTER(Dropout)],
    "db200_embed_bwd_ex": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_i64,
                           ctypes.POINTER(Dropout), ctypes.POINTER(Dropout)],
    "db200_dropout_mask": [c_vp, ctypes.POINTER(Dropout), c_int, c_i64, c_i64, c_i64, c_vp],
    "db200_assemble_tokens": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int],
    "db200_assemble_tokens_ex": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, ctypes.c_int32,
                                 ctypes.POINTER(Dropout)],
    "db200_assemble_tokens_pp": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, ctypes.c_int32, ctypes.c_int32,
                                 ctypes.POINTER(Dropout)],
    "db200_pos_compose": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int],
    "db200_pos_fold": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int],
    "db200_shift_labels": [c_vp, c_vp, c_vp, c_int, c_int, c_int],
    "db200_layernorm_fwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_f32],
    "db200_layernorm_residual_fwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_f32],
    "db200_layernorm_scale_residual_fwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_f32],
    "db200_layer_scale_residual_fwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int],
    "db200_layernorm_divmax_fwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_f32],
    "db200_layernorm_divmax_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int,
                                   c_int, c_vp, c_vp, c_i64],
    "db200_embed_bwd_scaled": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_i64, c_vp, c_vp,
                               c_f32],
    "db200_layer_scale_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int,
                              c_vp, c_i64],
    "db200_layernorm_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_i64],
    "db200_layernorm_bwd_ex": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp,
                               c_i64],
    "db200_layernorm_bwd_dropout": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int,
                                    c_int, ctypes.POINTER(Dropout), c_vp, c_i64],
    "db200_gemm_bf16": [c_vp, c_vp, c_int, c_i64, c_vp, c_int, c_i64, c_vp, c_i64, c_int, c_int, c_int,
                        ctypes.POINTER(GemmEpilogue)],
    "db200_gemm_bf16_ex": [c_vp, c_vp, c_int, c_i64, c_vp, c_int, c_i64, c_vp, c_i64, c_int, c_int, c_int,
                           ctypes.POINTER(GemmEpilogue), ctypes.POINTER(Dropout)],
    "db200_gemm_bf16_ce_weighted": [c_vp, c_vp, c_int, c_i64, c_vp, c_int, c_i64, c_vp, c_i64, c_int, c_int, c_int,
                                    ctypes.POINTER(GemmEpilogue), ctypes.POINTER(CeWeights)],
    "db200_gemm_bf16_gelu": [c_vp, c_vp, c_int, c_i64, c_vp, c_int, c_i64, c_vp, c_i64, c_int, c_int, c_int,
                             ctypes.POINTER(GemmEpilogue), c_vp, c_i64],
    "db200_gemm_bf16_gelu_bwd": [c_vp, c_vp, c_int, c_i64, c_vp, c_int, c_i64, c_vp, c_i64, c_int, c_int, c_int,
                                 ctypes.POINTER(GemmEpilogue)],
    "db200_gemm_bf16_glu": [c_vp, c_vp, c_int, c_i64, c_vp, c_int, c_i64, c_vp, c_i64, c_int, c_int, c_int,
                            ctypes.POINTER(GemmEpilogue), c_int, c_vp, c_i64],
    "db200_gemm_bf16_glu_bwd": [c_vp, c_vp, c_int, c_i64, c_vp, c_int, c_i64, c_vp, c_i64, c_int, c_int, c_int,
                                ctypes.POINTER(GemmEpilogue), c_int],
    "db200_gemm_ce_tiles": [c_int],
    "db200_embed_fwd_at": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_attn_decode": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_f32],
    "db200_sample_rows": [c_vp, c_vp, c_vp, c_vp, c_int, c_i64, c_int, c_int, c_f32],
    "db200_onehot_rows_f32": [c_vp, c_vp, c_vp, c_int, c_int, c_int],
    "db200_embed_fwd_at_dev": [c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp],
    "db200_attn_decode_dev": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_f32],
    "db200_attn_decode_local": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_f32],
    "db200_attn_decode_local_dev": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_int, c_f32],
    "db200_attn_decode_axial": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                c_f32],
    "db200_attn_decode_axial_dev": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int,
                                    c_f32],
    "db200_attn_decode_block_sparse": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int,
                                       c_f32],
    "db200_attn_decode_block_sparse_dev": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_int,
                                           c_f32],
    "db200_attn_decode_conv": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                               c_f32],
    "db200_attn_decode_conv_dev": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int,
                                   c_f32],
    "db200_sample_rows_at": [c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_i64, c_int, c_int, c_f32, c_vp],
    "db200_incr_i32": [c_vp, c_vp, c_int],
    "db200_sample_rows_filtered": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_i64, c_int, c_int, c_f32, c_int, c_f32],
    "db200_sample_rows_filtered_at": [c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_int, c_i64, c_int, c_int, c_f32, c_int,
                                      c_f32, c_vp],
    "db200_sample_rows_guided": [c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_int, c_int, c_int, c_f32, c_f32, c_int,
                                 c_f32, c_vp],
    "db200_caption_next": [c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_int, c_int, c_int, c_int, c_int, c_int],
    "db200_caption_next_at": [c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp],
    "db200_kv_cache_fill": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int],
    "db200_rows_repeat": [c_vp, c_vp, c_i64, c_vp, c_int, c_int, c_int],
    "db200_rope_fwd": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_rope_bwd": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_rope_decode": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int],
    "db200_rope_decode_dev": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp],
    "db200_rope_emb_fwd": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_rope_emb_bwd": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_rope_emb_decode": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int],
    "db200_rope_emb_decode_dev": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp],
    "db200_shift_tokens_fwd": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_shift_tokens_bwd": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_shift_tokens_decode": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int],
    "db200_shift_tokens_decode_dev": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp],
    "db200_shift_cache_fill": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_sgu_mix_fwd": [c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_int],
    "db200_sgu_mix_dgrad": [c_vp, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int],
    "db200_sgu_mix_wgrad": [c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_int, c_int],
    "db200_sgu_bwd": [c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_int, c_int, c_int],
    "db200_sgu_gate_bwd": [c_vp, c_vp, c_vp, c_i64, c_vp, c_i64, c_int, c_int],
    "db200_sgu_decode": [c_vp, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int],
    "db200_sgu_decode_dev": [c_vp, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp],
    "db200_sgu_cache_fill": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_crc32c": [c_vp, c_u64, c_vp],
    "db200_tfrecord_masked_crc": [c_vp, c_u64, c_vp],
    "db200_tfrecord_frame": [c_vp, c_u64, c_vp],
    "db200_tfrecord_index": [c_vp, c_u64, c_int, c_vp, c_vp, c_u64, c_vp],
    "db200_image_crop_resize_normalize": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int],
    "db200_ce_finish": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_i64],
    "db200_ce_finish_weighted": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, ctypes.POINTER(CeWeights),
                                 c_vp, c_i64],
    "db200_logits_mask_partition": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int,
                                    c_int, c_int, c_int],
    "db200_logits_mask_scatter": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int],
    "db200_attn_causal_fwd": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_f32],
    "db200_attn_causal_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_f32],
    "db200_attn_causal_fwd_ex": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_f32, ctypes.POINTER(Dropout)],
    "db200_attn_causal_bwd_ex": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_f32,
                                 ctypes.POINTER(Dropout)],
    "db200_attn_local_fwd": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_f32],
    "db200_attn_local_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_f32],
    "db200_attn_axial_fwd": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_f32],
    "db200_attn_axial_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int,
                             c_int, c_f32],
    "db200_attn_block_sparse_fwd": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_int, c_f32],
    "db200_attn_block_sparse_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp,
                                    c_int, c_f32],
    "db200_attn_conv_fwd": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_f32],
    "db200_attn_conv_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int,
                            c_int, c_f32],
    "db200_colsum_bf16": [c_vp, c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_i64],
    "db200_cast_f32_to_bf16": [c_vp, c_vp, c_vp, c_sz],
    "db200_cast_bf16_to_f32": [c_vp, c_vp, c_vp, c_sz],
    "db200_split_f32_to_bf16x2": [c_vp, c_vp, c_vp, c_vp, c_sz],
    "db200_sqnorm_f32": [c_vp, c_vp, c_sz, c_vp, c_vp, c_i64],
    "db200_adam_step": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_sz, c_f32, c_f32, c_f32, c_f32, c_f32, c_vp, c_f32,
                        c_f32, c_int, c_int, c_int],
    "db200_conv2d_fwd": [c_vp, ctypes.POINTER(ConvDesc), c_vp, c_vp, c_vp, c_vp, c_vp],
    "db200_conv2d_fwd_tc": [c_vp, ctypes.POINTER(ConvDesc), c_vp, c_vp, c_vp, c_vp, c_vp],
    "db200_conv2d_dgrad_tc": [c_vp, ctypes.POINTER(ConvDesc), c_vp, c_vp, c_vp, c_vp, c_vp],
    "db200_conv2d_wgrad_tc": [c_vp, ctypes.POINTER(ConvDesc), c_vp, c_vp, c_vp],
    "db200_conv2d_first_fwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int],
    "db200_conv2d_first_fwd_fma": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int],
    "db200_conv2d_dgrad": [c_vp, ctypes.POINTER(ConvDesc), c_vp, c_vp, c_vp, c_vp, c_vp],
    "db200_conv2d_wgrad": [c_vp, ctypes.POINTER(ConvDesc), c_vp, c_vp, c_vp, c_vp],
    "db200_conv7x7_in_fwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int],
    "db200_conv7x7_in_wgrad": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_i64],
    "db200_maxpool2x2_fwd": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_maxpool2x2_bwd": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_upsample2x_fwd": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_upsample2x_bwd": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_residual_gain": [c_vp, c_vp, c_vp, c_vp, c_f32, c_vp, c_vp, c_i64, c_int],
    "db200_rowmatmul_f32":[c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_rowmatmul_tn_f32": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int],
    "db200_gumbel_softmax_fwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_f32, c_int],
    "db200_gumbel_softmax_bwd": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_f32],
    "db200_argmax_rows_f32": [c_vp, c_vp, c_vp, c_int, c_int],
    "db200_groupnorm_stats": [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_f32, c_vp, c_i64],
    "db200_groupnorm_apply": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int],
    "db200_attn_noncausal_fwd": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_f32],
    "db200_attn_noncausal_long_fwd": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_f32],
    "db200_gather_rows_split": [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int],
    "db200_clamp_bf16_to_f32": [c_vp, c_vp, c_vp, c_i64, c_f32, c_f32],
    "db200_vae_kl_stats": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_f32, c_vp, c_i64],
    "db200_gumbel_softmax_bwd_kl": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_f32, c_f32],
    "db200_mse_fwd_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_sz, c_f32],
    "db200_logit_laplace_fwd_bwd": [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_f32, c_vp, c_i64],
    "db200_gather_cast_bf16_f32": [c_vp, c_vp, c_vp, c_vp, c_int],
    "db200_space_to_depth_f32": [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int],
    "db200_comm_load_nccl": [ctypes.c_char_p],
    "db200_comm_unique_id": [c_vp, c_sz],
    "db200_comm_create": [c_int, c_int, c_int, c_vp, c_int, ctypes.POINTER(c_vp)],
    "db200_comm_destroy": [c_vp],
    "db200_set_reserved_sms": [c_int],
    "db200_comm_register": [c_vp, c_vp, c_sz, ctypes.POINTER(c_int)],
    "db200_comm_info": [c_vp, ctypes.POINTER(c_int), ctypes.POINTER(c_int), ctypes.POINTER(c_int)],
    "db200_bucket_allreduce_launch": [c_vp, c_vp, c_vp, c_sz, c_int],
    "db200_bucket_reduce_scatter_launch": [c_vp, c_vp, c_vp, c_vp, c_sz, c_int],
    "db200_bucket_all_gather_launch": [c_vp, c_vp, c_vp, c_vp, c_sz, c_int],
    "db200_bucket_allreduce_wait": [c_vp, c_vp],
}
# scratch sizes of the ops whose reductions go through a caller-provided workspace (restype int64)
_WORKSPACE_QUERIES = {
    "db200_gemm_workspace_bytes": [c_int, c_int, c_int, ctypes.POINTER(GemmEpilogue)],
    "db200_layernorm_bwd_workspace_bytes": [c_int, c_int],
    "db200_layer_scale_bwd_workspace_bytes": [c_int, c_int],
    "db200_colsum_workspace_bytes": [c_int, c_int],
    "db200_sqnorm_workspace_bytes": [c_sz],
    "db200_ce_finish_workspace_bytes": [c_int],
    "db200_ce_finish_weighted_workspace_bytes": [c_int],
    "db200_embed_bwd_workspace_bytes": [c_int, c_int],
    "db200_vae_kl_stats_workspace_bytes": [c_int, c_int],
    "db200_logit_laplace_workspace_bytes": [c_i64, c_int],
    "db200_conv7x7_in_wgrad_workspace_bytes": [c_int, c_int, c_int, c_int, c_int],
    "db200_groupnorm_stats_workspace_bytes": [c_int, c_int, c_int, c_int],
}
EXPORTED_SYMBOLS = ["db200_last_error", "db200_launch_count"] + sorted(_SIGNATURES) + sorted(_WORKSPACE_QUERIES)

_lib = None
MISSING_SYMBOLS = []


class DB200Error(RuntimeError):
    pass


def load():
    """Load the shared object (once) and declare every prototype.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DB200Error(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / eager fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    lib.db200_last_error.restype = ctypes.c_char_p
    lib.db200_last_error.argtypes = []
    lib.db200_launch_count.restype = ctypes.c_ulonglong
    lib.db200_launch_count.argtypes = []
    for name, argtypes in _SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            MISSING_SYMBOLS.append(name)  # the CPU test-suite asserts this list is empty
            continue
        fn.argtypes = argtypes
        fn.restype = c_int
    for name, argtypes in _WORKSPACE_QUERIES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            MISSING_SYMBOLS.append(name)
            continue
        fn.argtypes = argtypes
        fn.restype = c_i64
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().db200_last_error().decode("utf-8", "replace")
        raise DB200Error(f"{what} failed with code {rc}: {msg}")


_device_ok = False


def require_device():
    """Fail loudly unless the current CUDA device can run the sm_90a cubins."""
    global _device_ok
    if _device_ok:
        return
    if not torch.cuda.is_available():
        raise DB200Error("CUDA device required: dalle_mtf_b200 has no CPU fallback")
    check(load().db200_device_check(), "db200_device_check")
    _device_ok = True


def launch_count():
    return int(load().db200_launch_count())


def stream_ptr():
    return torch.cuda.current_stream().cuda_stream


def workspace(nbytes):
    """Scratch for one call's ordered reductions, from PyTorch's caching allocator on the current stream (None if 0)."""
    if nbytes <= 0:
        return None
    return torch.empty(int(nbytes), dtype=torch.uint8, device=torch.cuda.current_device())


def ptr(t):
    """Device pointer of a tensor (None -> NULL).  The tensor must be contiguous in its last dimension."""
    if t is None:
        return None
    return t.data_ptr()
