"""Tensor-level wrappers over the C ABI (one Python function per exported kernel family).

Every function enqueues on torch's current CUDA stream and returns without synchronising.  Tensors are only
containers for device memory here; no torch arithmetic happens on the product path.
"""
import ctypes

import torch

from . import lib as L
from .lib import GemmEpilogue, ConvDesc, check, ptr, stream_ptr

BF16 = torch.bfloat16
F32 = torch.float32
I32 = torch.int32


def _chk(t, dtype, name):
    if t is None:
        return
    if not t.is_cuda:
        raise L.DB200Error(f"{name}: tensor must live on a CUDA device (no CPU fallback)")
    if t.dtype != dtype:
        raise L.DB200Error(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if t.dim() > 0 and t.stride(-1) != 1:
        raise L.DB200Error(f"{name}: innermost dimension must be contiguous")


# ----------------------------------------------------------------------------------------------- GEMM
# bench.py sets GEMM_PROFILE to a list to time every wgmma GEMM launch with CUDA events on the launching stream:
# entries are (start_event, end_event, algorithmic_flops).
GEMM_PROFILE = None


def _nbytes(ws):
    return ws.numel() if ws is not None else 0


def gemm(a, b, out, M, N, K, *, a_mn=False, b_mn=False, lda=None, ldb=None, ldd=None, mode=L.EPI_STORE,
         alpha=1.0, bias=None, relu=False, residual=None, aux=None, split_k=1, labels=None, part_max=None,
         part_sum=None, label_logit=None, lse=None, n_valid=0, colsum=None):
    """D[M,N] = A[M,K] @ B[K,N] on wgmma.  a_mn / b_mn: operand is stored with M (resp. N) contiguous.

    a: [M,K] (k-major) or [K,M] (mn-major);  b: [N,K] (k-major) or [K,N] (mn-major).
    """
    L.require_device()
    _chk(a, BF16, "gemm A")
    _chk(b, BF16, "gemm B")
    lda = lda if lda is not None else a.stride(0)
    ldb = ldb if ldb is not None else b.stride(0)
    e = GemmEpilogue()
    e.mode = mode
    e.out_f32 = 1 if (out is not None and out.dtype == F32) else 0
    e.relu = 1 if relu else 0
    e.split_k = split_k
    e.alpha = alpha
    _chk(bias, F32, "gemm bias")
    e.bias = ptr(bias)
    _chk(residual, BF16, "gemm residual")
    e.residual = ptr(residual)
    e.ldr = residual.stride(0) if residual is not None else 0
    _chk(aux, BF16, "gemm aux")
    e.aux = ptr(aux)
    e.ldaux = aux.stride(0) if aux is not None else 0
    _chk(labels, I32, "gemm labels")
    e.labels = ptr(labels)
    e.part_max, e.part_sum, e.label_logit, e.lse = ptr(part_max), ptr(part_sum), ptr(label_logit), ptr(lse)
    e.n_valid = n_valid
    _chk(colsum, F32, "gemm colsum")
    e.colsum = ptr(colsum)
    if out is not None:
        if mode == L.EPI_ATOMIC:
            _chk(out, F32, "gemm D (atomic)")
        ldd = ldd if ldd is not None else out.stride(0)
    else:
        ldd = 0
    ws = L.workspace(L.load().db200_gemm_workspace_bytes(M, N, K, ctypes.byref(e)))
    e.workspace, e.workspace_bytes = ptr(ws), (ws.numel() if ws is not None else 0)
    prof = GEMM_PROFILE
    if prof is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
    check(L.load().db200_gemm_bf16(stream_ptr(), ptr(a), int(a_mn), lda, ptr(b), int(b_mn), ldb, ptr(out), ldd,
                                   M, N, K, ctypes.byref(e)), "db200_gemm_bf16")
    if prof is not None:
        ev1.record()
        prof.append((ev0, ev1, 2.0 * M * N * K, (M, N, K, mode, int(a_mn), int(b_mn))))
    return out


def linear_fwd(x, w, out, bias=None, relu=False, residual=None):
    """out[T,N] = act(x[T,K] @ w[K,N] + bias) + residual      (forward: A k-major, B mn-major)."""
    T, K = x.shape
    N = w.shape[1]
    return gemm(x, w, out, T, N, K, a_mn=False, b_mn=True, bias=bias, relu=relu, residual=residual)


def linear_dgrad(dy, w, out, relu_mask_of=None, colsum=None):
    """out[T,K] = dy[T,N] @ w[K,N]^T  (optionally masked by relu_mask_of > 0; colsum[k] += sum_t out[t,k])."""
    T, N = dy.shape
    K = w.shape[0]
    if relu_mask_of is not None:
        return gemm(dy, w, out, T, K, N, a_mn=False, b_mn=False, mode=L.EPI_RELU_BWD, aux=relu_mask_of, colsum=colsum)
    return gemm(dy, w, out, T, K, N, a_mn=False, b_mn=False)


def linear_wgrad(x, dy, dw, N=None):
    """dw[K,N] (f32) += x[T,K]^T @ dy[T,N]      (both operands mn-major, split-K summed in split order)."""
    T, K = x.shape
    N = N if N is not None else dy.shape[1]
    return gemm(x, dy, dw, K, N, T, a_mn=True, b_mn=True, mode=L.EPI_ATOMIC, split_k=0)


def ce_tiles(N):
    return L.load().db200_gemm_ce_tiles(N)


def ce_finish(part_max, part_sum, label_logit, lse, loss_rows, loss_sum):
    L.require_device()
    n_tiles, M = part_max.shape          # tile-major partials [n_tiles][M]
    ws = L.workspace(L.load().db200_ce_finish_workspace_bytes(M))
    check(L.load().db200_ce_finish(stream_ptr(), ptr(part_max), ptr(part_sum), ptr(label_logit), ptr(lse),
                                   ptr(loss_rows), ptr(loss_sum), M, n_tiles, ptr(ws), _nbytes(ws)),
          "db200_ce_finish")


# ----------------------------------------------------------------------------------------------- row ops
def embed_fwd(ids, wte, wpe, out):
    L.require_device()
    _chk(ids, I32, "ids"); _chk(wte, BF16, "wte"); _chk(wpe, BF16, "wpe"); _chk(out, BF16, "out")
    B, S = ids.shape
    V, d = wte.shape
    check(L.load().db200_embed_fwd(stream_ptr(), ptr(ids), ptr(wte), ptr(wpe), ptr(out), B, S, d, V), "embed_fwd")
    return out


def embed_bwd(ids, dx, dwte, dwpe):
    L.require_device()
    _chk(ids, I32, "ids"); _chk(dx, BF16, "dx"); _chk(dwte, F32, "dwte"); _chk(dwpe, F32, "dwpe")
    B, S = ids.shape
    V, d = dwte.shape
    ws = L.workspace(L.load().db200_embed_bwd_workspace_bytes(d, V))
    check(L.load().db200_embed_bwd(stream_ptr(), ptr(ids), ptr(dx), ptr(dwte), ptr(dwpe), B, S, d, V, ptr(ws),
                                   _nbytes(ws)), "embed_bwd")


def assemble_tokens(text_ids, image_idx, tokens, image_offset):
    L.require_device()
    _chk(text_ids, I32, "text_ids"); _chk(image_idx, I32, "image_idx"); _chk(tokens, I32, "tokens")
    B, Tt = text_ids.shape
    Ti = image_idx.shape[1]
    check(L.load().db200_assemble_tokens(stream_ptr(), ptr(text_ids), ptr(image_idx), ptr(tokens), B, Tt, Ti,
                                         image_offset), "assemble_tokens")
    return tokens


def shift_labels(ids, labels, eos_id):
    L.require_device()
    _chk(ids, I32, "ids"); _chk(labels, I32, "labels")
    B, S = ids.shape
    check(L.load().db200_shift_labels(stream_ptr(), ptr(ids), ptr(labels), B, S, eos_id), "shift_labels")
    return labels


def layernorm_fwd(x, g, b, y, mean, rstd, eps=1e-5):
    L.require_device()
    _chk(x, BF16, "x"); _chk(y, BF16, "y"); _chk(g, F32, "g"); _chk(b, F32, "b")
    _chk(mean, F32, "mean"); _chk(rstd, F32, "rstd")
    rows, d = x.shape
    check(L.load().db200_layernorm_fwd(stream_ptr(), ptr(x), ptr(g), ptr(b), ptr(y), ptr(mean), ptr(rstd), rows, d,
                                       eps), "layernorm_fwd")
    return y


def layernorm_bwd(dy, x, g, mean, rstd, dres, dx, dg, db, dxsum=None):
    """dxsum (optional, f32 [d]): += column sums of the produced dx (fused bias gradient of the layer below)."""
    L.require_device()
    _chk(dy, BF16, "dy"); _chk(x, BF16, "x"); _chk(dres, BF16, "dres"); _chk(dx, BF16, "dx")
    _chk(g, F32, "g"); _chk(dg, F32, "dg"); _chk(db, F32, "db"); _chk(dxsum, F32, "dxsum")
    rows, d = x.shape
    ws = L.workspace(L.load().db200_layernorm_bwd_workspace_bytes(rows, d))
    check(L.load().db200_layernorm_bwd_ex(stream_ptr(), ptr(dy), ptr(x), ptr(g), ptr(mean), ptr(rstd), ptr(dres),
                                          ptr(dx), ptr(dg), ptr(db), ptr(dxsum), rows, d, ptr(ws), _nbytes(ws)),
          "layernorm_bwd")
    return dx


def colsum(x, out_accum, rows=None, cols=None):
    L.require_device()
    _chk(x, BF16, "x"); _chk(out_accum, F32, "out_accum")
    rows = rows if rows is not None else x.shape[0]
    cols = cols if cols is not None else x.shape[1]
    ws = L.workspace(L.load().db200_colsum_workspace_bytes(rows, cols))
    check(L.load().db200_colsum_bf16(stream_ptr(), ptr(x), x.stride(0), rows, cols, ptr(out_accum), ptr(ws),
                                     _nbytes(ws)), "colsum")


def cast_f32_to_bf16(src, dst):
    L.require_device()
    _chk(src, F32, "src"); _chk(dst, BF16, "dst")
    check(L.load().db200_cast_f32_to_bf16(stream_ptr(), ptr(src), ptr(dst), src.numel()), "cast_f32_to_bf16")
    return dst


def cast_bf16_to_f32(src, dst):
    L.require_device()
    _chk(src, BF16, "src"); _chk(dst, F32, "dst")
    check(L.load().db200_cast_bf16_to_f32(stream_ptr(), ptr(src), ptr(dst), src.numel()), "cast_bf16_to_f32")
    return dst


def split_f32(src, hi, lo=None):
    """hi = bf16(src), lo = bf16(src - hi)."""
    L.require_device()
    _chk(src, F32, "src"); _chk(hi, BF16, "hi"); _chk(lo, BF16, "lo")
    check(L.load().db200_split_f32_to_bf16x2(stream_ptr(), ptr(src), ptr(hi), ptr(lo), src.numel()), "split_f32")


# ----------------------------------------------------------------------------------------------- attention
# bench.py sets ATTN_PROFILE to a list to time every attention launch like GEMM_PROFILE: entries are
# (start_event, end_event, causal-algorithmic flops, "fwd" | "bwd").  Forward = 2 products over the visible half of the
# S x S logits: 4 S^2 dh B H / 2; backward = 2.5 x that (5 products).
ATTN_PROFILE = None


def _attn_timed(kind, B, S, H, dh, call):
    prof = ATTN_PROFILE
    if prof is None:
        return call()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    call()
    ev1.record()
    prof.append((ev0, ev1, 2.0 * S * S * dh * B * H * (1.0 if kind == "fwd" else 2.5), kind))


def attn_fwd(qkv, out, lse, B, S, H, dh, scale=1.0):
    L.require_device()
    _chk(qkv, BF16, "qkv"); _chk(out, BF16, "out"); _chk(lse, F32, "lse")
    _attn_timed("fwd", B, S, H, dh, lambda: check(
        L.load().db200_attn_causal_fwd(stream_ptr(), ptr(qkv), ptr(out), ptr(lse), B, S, H, dh, scale),
        "attn_causal_fwd"))
    return out


def attn_bwd(qkv, out, dout, lse, dq_accum, delta, dqkv, B, S, H, dh, scale=1.0):
    L.require_device()
    _chk(qkv, BF16, "qkv"); _chk(out, BF16, "out"); _chk(dout, BF16, "dout"); _chk(dqkv, BF16, "dqkv")
    _chk(lse, F32, "lse"); _chk(dq_accum, F32, "dq_accum"); _chk(delta, F32, "delta")
    _attn_timed("bwd", B, S, H, dh, lambda: check(
        L.load().db200_attn_causal_bwd(stream_ptr(), ptr(qkv), ptr(out), ptr(dout), ptr(lse), ptr(dq_accum),
                                       ptr(delta), ptr(dqkv), B, S, H, dh, scale), "attn_causal_bwd"))
    return dqkv


# ----------------------------------------------------------------------------------------------- optimiser
def sqnorm(g, out_accum):
    L.require_device()
    _chk(g, F32, "g"); _chk(out_accum, F32, "out_accum")
    ws = L.workspace(L.load().db200_sqnorm_workspace_bytes(g.numel()))
    check(L.load().db200_sqnorm_f32(stream_ptr(), ptr(g), g.numel(), ptr(out_accum), ptr(ws), _nbytes(ws)), "sqnorm")


def adam_step(p, m, v, g, p_bf16, lr, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.0, gnorm_sq=None,
              clip=0.0, grad_scale=1.0, bias_correction=False, step=0, zero_grad=False):
    L.require_device()
    for t, n in ((p, "p"), (m, "m"), (v, "v"), (g, "g")):
        _chk(t, F32, n)
    _chk(p_bf16, BF16, "p_bf16")
    check(L.load().db200_adam_step(stream_ptr(), ptr(p), ptr(m), ptr(v), ptr(g), ptr(p_bf16), p.numel(), lr, beta1,
                                   beta2, eps, weight_decay, ptr(gnorm_sq), clip, grad_scale, int(bias_correction),
                                   int(step), int(zero_grad)), "adam_step")


# ----------------------------------------------------------------------------------------------- VAE ops
def conv_desc(N, H, W, Cin, Cout, KH, KW, stride, transposed=False, act_f32=True, relu=False):
    c = ConvDesc()
    c.N, c.H, c.W, c.Cin, c.Cout = N, H, W, Cin, Cout
    c.KH, c.KW, c.stride = KH, KW, stride
    if transposed:
        c.Ho, c.Wo = H * stride, W * stride
    else:
        c.Ho, c.Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    c.transposed = int(transposed)
    c.act_f32 = int(act_f32)
    c.relu = int(relu)
    return c


def gather_cast(src_bf16, dst_f32, table_dev, n_segments):
    L.require_device()
    check(L.load().db200_gather_cast_bf16_f32(stream_ptr(), ptr(src_bf16), ptr(dst_f32), ptr(table_dev), n_segments),
          "gather_cast")


def space_to_depth(x, out, s, inverse=False):
    """tf.space_to_depth / depth_to_space on f32 NHWC.  `x` is the flat image [N,H,W,C] (inverse: the deep one)."""
    L.require_device()
    flat = out if inverse else x
    N, H, W, C = flat.shape
    check(L.load().db200_space_to_depth_f32(stream_ptr(), ptr(x), ptr(out), N, H, W, C, int(s), int(inverse)),
          "space_to_depth")
    return out


def conv2d_fwd(c, x, w, bias, residual, y):
    L.require_device()
    check(L.load().db200_conv2d_fwd(stream_ptr(), ctypes.byref(c), ptr(x), ptr(w), ptr(bias), ptr(residual),
                                    ptr(y)), "conv2d_fwd")
    return y


def conv2d_fwd_tc(c, x, w_bf16, bias, residual, y):
    """wgmma implicit-GEMM forward (bf16 activations / kernel).  Raises if the shape is not supported."""
    L.require_device()
    _chk(x, BF16, "x"); _chk(w_bf16, BF16, "w"); _chk(y, BF16, "y"); _chk(residual, BF16, "residual")
    check(L.load().db200_conv2d_fwd_tc(stream_ptr(), ctypes.byref(c), ptr(x), ptr(w_bf16), ptr(bias), ptr(residual),
                                       ptr(y)), "conv2d_fwd_tc")
    return y


def conv2d_first_fwd(x_f32, w, bias, y_bf16):
    """First encoder layer: fp32 image [N,H,W,3] -> bf16 [N,H/2,W/2,Cout] (4x4, stride 2, SAME)."""
    L.require_device()
    _chk(x_f32, F32, "x"); _chk(w, F32, "w"); _chk(bias, F32, "bias"); _chk(y_bf16, BF16, "y")
    N, H, W_, _ = x_f32.shape
    check(L.load().db200_conv2d_first_fwd(stream_ptr(), ptr(x_f32), ptr(w), ptr(bias), ptr(y_bf16), N, H, W_,
                                          w.shape[-1]), "conv2d_first_fwd")
    return y_bf16


def _tc_geometry_ok(c):
    if c.act_f32 or c.KH * c.KW > 16:
        return False
    if c.transposed:
        return c.KH == 4 and c.KW == 4 and c.stride == 2
    return c.stride == 1 or (c.stride == 2 and c.H % 2 == 0 and c.W % 2 == 0)


def conv_tc_supported(c):
    """forward (conv or conv-transpose) on wgmma"""
    return _tc_geometry_ok(c) and c.Cin % 64 == 0 and c.Cout % 8 == 0


def conv_dgrad_tc_supported(c):
    return _tc_geometry_ok(c) and c.Cout % 64 == 0 and c.Cin % 8 == 0


def conv_wgrad_tc_supported(c):
    return _tc_geometry_ok(c) and c.Cin % 64 == 0 and c.Cout % 64 == 0


def conv2d_dgrad_tc(c, dy, w_bf16, x_mask, dres, dx):
    L.require_device()
    _chk(dy, BF16, "dy"); _chk(w_bf16, BF16, "w"); _chk(x_mask, BF16, "x_mask"); _chk(dres, BF16, "dres"); _chk(dx, BF16, "dx")
    check(L.load().db200_conv2d_dgrad_tc(stream_ptr(), ctypes.byref(c), ptr(dy), ptr(w_bf16), ptr(x_mask), ptr(dres),
                                         ptr(dx)), "conv2d_dgrad_tc")
    return dx


def conv2d_wgrad_tc(c, x, dy, dw):
    L.require_device()
    _chk(x, BF16, "x"); _chk(dy, BF16, "dy"); _chk(dw, F32, "dw")
    check(L.load().db200_conv2d_wgrad_tc(stream_ptr(), ctypes.byref(c), ptr(x), ptr(dy), ptr(dw)), "conv2d_wgrad_tc")


def conv2d_dgrad(c, dy, w, x_mask, dres, dx):
    L.require_device()
    check(L.load().db200_conv2d_dgrad(stream_ptr(), ctypes.byref(c), ptr(dy), ptr(w), ptr(x_mask), ptr(dres),
                                      ptr(dx)), "conv2d_dgrad")
    return dx


def conv2d_wgrad(c, x, dy, dw, dbias):
    L.require_device()
    check(L.load().db200_conv2d_wgrad(stream_ptr(), ctypes.byref(c), ptr(x), ptr(dy), ptr(dw), ptr(dbias)),
          "conv2d_wgrad")


def rowmatmul(a, b, out, rows, K, N, b_transposed=False, accumulate=False):
    L.require_device()
    check(L.load().db200_rowmatmul_f32(stream_ptr(), ptr(a), ptr(b), ptr(out), rows, K, N, int(b_transposed),
                                       int(accumulate)), "rowmatmul")
    return out


def rowmatmul_tn(a, b, out_accum, rows, M, N):
    L.require_device()
    check(L.load().db200_rowmatmul_tn_f32(stream_ptr(), ptr(a), ptr(b), ptr(out_accum), rows, M, N), "rowmatmul_tn")


def gumbel_softmax_fwd(logits, u, y_soft, y_out, idx, rows, K, tau, hard):
    L.require_device()
    check(L.load().db200_gumbel_softmax_fwd(stream_ptr(), ptr(logits), ptr(u), ptr(y_soft), ptr(y_out), ptr(idx),
                                            rows, K, tau, int(hard)), "gumbel_softmax_fwd")


def gumbel_softmax_bwd(y_soft, dy, dlogits, rows, K, tau):
    L.require_device()
    check(L.load().db200_gumbel_softmax_bwd(stream_ptr(), ptr(y_soft), ptr(dy), ptr(dlogits), rows, K, tau),
          "gumbel_softmax_bwd")


def argmax_rows(x, idx, rows, K):
    L.require_device()
    check(L.load().db200_argmax_rows_f32(stream_ptr(), ptr(x), ptr(idx), rows, K), "argmax_rows")


def mse_fwd_bwd(pred, target, dpred, loss_accum, scale):
    L.require_device()
    check(L.load().db200_mse_fwd_bwd(stream_ptr(), ptr(pred), ptr(target), ptr(dpred), ptr(loss_accum),
                                     pred.numel(), scale), "mse_fwd_bwd")


# ----------------------------------------------------------------------------------------------- input pipeline (N2)
def image_crop_resize_normalize(packed_u8, offsets_i64, heights_i32, widths_i32, boxes_f32, out_f32, channels, size):
    """decode_img's crop_and_resize + (x - 127.5) / 127.5 for a packed batch of decoded uint8 images (input_fns.py:4-21)."""
    L.require_device()
    _chk(packed_u8, torch.uint8, "packed"); _chk(offsets_i64, torch.int64, "offsets")
    _chk(heights_i32, torch.int32, "heights"); _chk(widths_i32, torch.int32, "widths")
    _chk(boxes_f32, F32, "boxes"); _chk(out_f32, F32, "out")
    B = heights_i32.numel()
    assert out_f32.shape == (B, size, size, channels) and boxes_f32.shape == (B, 4)
    check(L.load().db200_image_crop_resize_normalize(stream_ptr(), ptr(packed_u8), ptr(offsets_i64), ptr(heights_i32),
                                                     ptr(widths_i32), ptr(boxes_f32), ptr(out_f32), B, channels, size),
          "db200_image_crop_resize_normalize")
    return out_f32


# ----------------------------------------------------------------------------------------------- decoding (N4)
def embed_fwd_at(ids, wte, wpe, out, pos):
    """x[b,:] = wte[ids[b]] + wpe[pos]   (models.py:186-219 at one position)."""
    L.require_device()
    _chk(ids, I32, "ids"); _chk(wte, BF16, "wte"); _chk(wpe, BF16, "wpe"); _chk(out, BF16, "out")
    B, d = out.shape
    check(L.load().db200_embed_fwd_at(stream_ptr(), ptr(ids), ptr(wte), ptr(wpe), ptr(out), B, d, wte.shape[0],
                                      wpe.shape[0], int(pos)), "db200_embed_fwd_at")
    return out


def attn_decode(qkv_step, k_cache, v_cache, out, pos, scale):
    """Append this position's k, v to the caches and attend with its q over keys <= pos (models.py:246-254, 281-299)."""
    L.require_device()
    _chk(qkv_step, BF16, "qkv_step"); _chk(k_cache, BF16, "k_cache"); _chk(v_cache, BF16, "v_cache"); _chk(out, BF16, "out")
    B, S, H, dh = k_cache.shape
    assert v_cache.shape == k_cache.shape and qkv_step.numel() == B * 3 * H * dh and out.numel() == B * H * dh
    check(L.load().db200_attn_decode(stream_ptr(), ptr(qkv_step), ptr(k_cache), ptr(v_cache), ptr(out), B, S, H, dh,
                                     int(pos), float(scale)), "db200_attn_decode")
    return out


def sample_rows(logits, u, idx, lo, hi, inv_temp=1.0):
    """idx[r] = lo + argmax over [lo, hi) of logits * inv_temp + Gumbel(u); u None = greedy (first maximum)."""
    L.require_device()
    _chk(logits, F32, "logits"); _chk(u, F32, "u"); _chk(idx, I32, "idx")
    rows = logits.shape[0]
    if u is not None:
        assert u.shape == (rows, hi - lo)
    check(L.load().db200_sample_rows(stream_ptr(), ptr(logits), ptr(u), ptr(idx), rows, logits.stride(0), int(lo),
                                     int(hi), float(inv_temp)), "db200_sample_rows")
    return idx


def embed_fwd_at_dev(tokens, wte, wpe, out, pos_dev):
    """embed_fwd_at with the position (and the token column) taken from the device scalar pos_dev (graph replay)."""
    L.require_device()
    _chk(tokens, I32, "tokens"); _chk(wte, BF16, "wte"); _chk(wpe, BF16, "wpe"); _chk(out, BF16, "out")
    B, d = out.shape
    check(L.load().db200_embed_fwd_at_dev(stream_ptr(), ptr(tokens), tokens.stride(0), ptr(wte), ptr(wpe), ptr(out), B,
                                          d, wte.shape[0], ptr(pos_dev)), "db200_embed_fwd_at_dev")
    return out


def attn_decode_dev(qkv_step, k_cache, v_cache, out, pos_dev, scale):
    L.require_device()
    B, S, H, dh = k_cache.shape
    check(L.load().db200_attn_decode_dev(stream_ptr(), ptr(qkv_step), ptr(k_cache), ptr(v_cache), ptr(out), B, S, H, dh,
                                         ptr(pos_dev), float(scale)), "db200_attn_decode_dev")
    return out


def sample_rows_at(logits, u, tokens, lo, hi, inv_temp, pos_dev):
    """tokens[r, pos + 1] = lo + argmax over [lo, hi) of logits * inv_temp + Gumbel(u)   (pos read on the device)."""
    L.require_device()
    _chk(logits, F32, "logits"); _chk(u, F32, "u"); _chk(tokens, I32, "tokens")
    check(L.load().db200_sample_rows_at(stream_ptr(), ptr(logits), ptr(u), ptr(tokens), tokens.stride(0),
                                        logits.shape[0], logits.stride(0), int(lo), int(hi), float(inv_temp),
                                        ptr(pos_dev)), "db200_sample_rows_at")
    return tokens


def incr_i32(p, delta=1):
    L.require_device()
    check(L.load().db200_incr_i32(stream_ptr(), ptr(p), int(delta)), "db200_incr_i32")


def onehot_rows(idx, y, offset=0):
    L.require_device()
    _chk(idx, I32, "idx"); _chk(y, F32, "y")
    rows, K = y.shape
    check(L.load().db200_onehot_rows_f32(stream_ptr(), ptr(idx), ptr(y), rows, K, int(offset)), "db200_onehot_rows_f32")
    return y
