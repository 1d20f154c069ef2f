"""Tensor-level wrappers over the C ABI (one Python function per exported kernel family).

Every function enqueues on torch's current CUDA stream and returns without synchronising.  Tensors are only
containers for device memory here; no torch arithmetic happens on the product path.
"""
import ctypes
import numbers

import torch

from . import lib as L
from .lib import GemmEpilogue, ConvDesc, check, ptr, stream_ptr


def _ref(d):
    """ctypes argument of an optional db200_dropout (None -> NULL)."""
    return ctypes.byref(d) if d is not None else None

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
    # a length-1 innermost dimension has no step to take: torch keeps any stride there (out[:, j].contiguous() of a
    # one-row [1, S] matrix is a view with stride S), and the kernels never apply it
    if t.dim() > 0 and t.stride(-1) != 1 and t.shape[-1] > 1:
        raise L.DB200Error(f"{name}: innermost dimension must be contiguous")


# ----------------------------------------------------------------------------------------------- GEMM
# bench.py sets GEMM_PROFILE to a list to time every wgmma GEMM launch with CUDA events on the launching stream:
# entries are (start_event, end_event, algorithmic_flops).
GEMM_PROFILE = None


def _nbytes(ws):
    return ws.numel() if ws is not None else 0


def gemm(a, b, out, M, N, K, *, a_mn=False, b_mn=False, lda=None, ldb=None, ldd=None, mode=L.EPI_STORE,
         alpha=1.0, bias=None, relu=False, residual=None, aux=None, split_k=1, labels=None, part_max=None,
         part_sum=None, label_logit=None, lse=None, n_valid=0, colsum=None, dropout=None, ce_weights=None, gelu=None,
         z=None, glu=None, glu_act=None):
    """D[M,N] = A[M,K] @ B[K,N] on wgmma.  a_mn / b_mn: operand is stored with M (resp. N) contiguous.

    a: [M,K] (k-major) or [K,M] (mn-major);  b: [N,K] (k-major) or [K,N] (mn-major).
    dropout (lib.Dropout, STORE only): D = residual + keep * scale * act(alpha * acc + bias).
    ce_weights (lib.CeWeights, CE_GRAD only, a k-major / b mn-major): the weighted CE_GRAD epilogue, which takes its
    per-row coefficients from the descriptor instead of alpha.
    gelu "fwd" (STORE, a k-major / b mn-major): D = gelu(bf16(alpha * acc + bias)), and z (bf16, or None) receives the
    rounded pre-activation; gelu "bwd" (RELU_BWD, both k-major): D = alpha * acc * gelu'(aux), aux = the stored z.
    glu "fwd" / "bwd" with glu_act "relu" or "gelu": the gated MLP's W1 store (STORE, a k-major / b mn-major, b = the
    [K, 2N] value | gate weight, N the width of D = h; z [M, 2N] or None) and its dgrad (RELU_BWD, both k-major, N the
    width of dh, D [M, 2N], aux = the stored z, colsum 2N entries); include/dalle_b200.h states their arithmetic.
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
    _chk(z, BF16, "gemm z")
    if z is not None and gelu != "fwd" and glu != "fwd":
        raise L.DB200Error("gemm: a pre-activation output needs the GELU or GLU forward epilogue")
    if glu is not None and (gelu is not None or glu not in ("fwd", "bwd") or glu_act not in ("relu", "gelu")):
        raise ValueError(f"gemm: glu must be 'fwd' or 'bwd' with glu_act 'relu' or 'gelu' and no gelu, got "
                         f"{glu!r}, {glu_act!r}, gelu={gelu!r}")
    e.colsum = ptr(colsum)
    if out is not None:
        if mode == L.EPI_ATOMIC:
            _chk(out, F32, "gemm D (atomic)")
        ldd = ldd if ldd is not None else out.stride(0)
    else:
        ldd = 0
    # the GLU backward's fused column sums span its 2N output columns
    ws = L.workspace(L.load().db200_gemm_workspace_bytes(M, 2 * N if glu == "bwd" else N, K, ctypes.byref(e)))
    e.workspace, e.workspace_bytes = ptr(ws), (ws.numel() if ws is not None else 0)
    prof = GEMM_PROFILE
    if prof is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
    if glu is not None:
        act = L.ACT_GELU if glu_act == "gelu" else L.ACT_RELU
        if glu == "fwd":
            check(L.load().db200_gemm_bf16_glu(stream_ptr(), ptr(a), int(a_mn), lda, ptr(b), int(b_mn), ldb, ptr(out),
                                               ldd, M, N, K, ctypes.byref(e), act, ptr(z),
                                               z.stride(0) if z is not None else 0), "db200_gemm_bf16_glu")
        else:
            check(L.load().db200_gemm_bf16_glu_bwd(stream_ptr(), ptr(a), int(a_mn), lda, ptr(b), int(b_mn), ldb,
                                                   ptr(out), ldd, M, N, K, ctypes.byref(e), act),
                  "db200_gemm_bf16_glu_bwd")
    elif gelu == "fwd":
        check(L.load().db200_gemm_bf16_gelu(stream_ptr(), ptr(a), int(a_mn), lda, ptr(b), int(b_mn), ldb, ptr(out),
                                            ldd, M, N, K, ctypes.byref(e), ptr(z), z.stride(0) if z is not None else 0),
              "db200_gemm_bf16_gelu")
    elif gelu == "bwd":
        check(L.load().db200_gemm_bf16_gelu_bwd(stream_ptr(), ptr(a), int(a_mn), lda, ptr(b), int(b_mn), ldb, ptr(out),
                                                ldd, M, N, K, ctypes.byref(e)), "db200_gemm_bf16_gelu_bwd")
    elif gelu is not None:
        raise ValueError(f"gemm: gelu must be None, 'fwd' or 'bwd', got {gelu!r}")
    elif ce_weights is not None:
        check(L.load().db200_gemm_bf16_ce_weighted(stream_ptr(), ptr(a), int(a_mn), lda, ptr(b), int(b_mn), ldb,
                                                   ptr(out), ldd, M, N, K, ctypes.byref(e), ctypes.byref(ce_weights)),
              "db200_gemm_bf16_ce_weighted")
    elif dropout is None:
        check(L.load().db200_gemm_bf16(stream_ptr(), ptr(a), int(a_mn), lda, ptr(b), int(b_mn), ldb, ptr(out), ldd,
                                       M, N, K, ctypes.byref(e)), "db200_gemm_bf16")
    else:
        check(L.load().db200_gemm_bf16_ex(stream_ptr(), ptr(a), int(a_mn), lda, ptr(b), int(b_mn), ldb, ptr(out),
                                          ldd, M, N, K, ctypes.byref(e), ctypes.byref(dropout)), "db200_gemm_bf16_ex")
    if prof is not None:
        ev1.record()
        prof.append((ev0, ev1, 2.0 * M * N * K, (M, N, K, mode, int(a_mn), int(b_mn))))
    return out


def linear_fwd(x, w, out, bias=None, relu=False, residual=None, dropout=None, gelu=False, z_out=None, glu=None):
    """out[T,N] = dropout(act(x[T,K] @ w[K,N] + bias)) + residual      (forward: A k-major, B mn-major).

    gelu: out = gelu(z) with z = bf16(x @ w + bias) (mtf's tanh GELU, no residual or dropout); z_out [T,N] bf16
    receives z for the backward, or is None (inference).
    glu "relu" / "gelu" (the gated MLP): w is [K, 2N'] and z = bf16(x @ w + bias) = [zv | zg]; out [T, N'] =
    bf16(zv * bf16(act(zg))); z_out [T, 2N'] receives z, or is None."""
    T, K = x.shape
    N = w.shape[1]
    if glu is not None:
        if relu or gelu or residual is not None or dropout is not None:
            raise L.DB200Error("linear_fwd: the GLU epilogue takes no relu, gelu, residual or dropout")
        if N % 2:
            raise L.DB200Error(f"linear_fwd: a GLU weight holds value and gate columns: even width, got {N}")
        return gemm(x, w, out, T, N // 2, K, a_mn=False, b_mn=True, bias=bias, glu="fwd", glu_act=glu, z=z_out)
    if gelu:
        if relu or residual is not None or dropout is not None:
            raise L.DB200Error("linear_fwd: the GELU epilogue takes no relu, residual or dropout")
        return gemm(x, w, out, T, N, K, a_mn=False, b_mn=True, bias=bias, gelu="fwd", z=z_out)
    if z_out is not None:
        raise L.DB200Error("linear_fwd: z_out needs gelu=True or glu")
    return gemm(x, w, out, T, N, K, a_mn=False, b_mn=True, bias=bias, relu=relu, residual=residual, dropout=dropout)


def linear_dgrad(dy, w, out, relu_mask_of=None, colsum=None, gelu_grad_of=None, glu_grad_of=None, glu=None):
    """out[T,K] = dy[T,N] @ w[K,N]^T  (optionally masked by relu_mask_of > 0, or multiplied by gelu'(gelu_grad_of),
    the stored pre-activation z; colsum[k] += sum_t out[t,k]).

    glu_grad_of = the stored z [T, 2K] of a gated MLP and glu = its nonlinearity ("relu" / "gelu"): dh = dy @ w^T is
    the gradient of h and out [T, 2K] receives [dzv | dzg] (include/dalle_b200.h), colsum 2K entries."""
    T, N = dy.shape
    K = w.shape[0]
    if sum(v is not None for v in (relu_mask_of, gelu_grad_of, glu_grad_of)) > 1:
        raise L.DB200Error("linear_dgrad: relu_mask_of, gelu_grad_of and glu_grad_of are exclusive")
    if (glu_grad_of is None) != (glu is None):
        raise L.DB200Error("linear_dgrad: glu_grad_of and glu go together")
    if glu_grad_of is not None:
        return gemm(dy, w, out, T, K, N, a_mn=False, b_mn=False, mode=L.EPI_RELU_BWD, aux=glu_grad_of,
                    colsum=colsum, glu="bwd", glu_act=glu)
    if gelu_grad_of is not None:
        return gemm(dy, w, out, T, K, N, a_mn=False, b_mn=False, mode=L.EPI_RELU_BWD, aux=gelu_grad_of,
                    colsum=colsum, gelu="bwd")
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


def ce_finish_weighted(part_max, part_sum, label_logit, lse, loss_rows, sums, weights):
    """Weighted finish (lib.CeWeights): loss_rows = CE + z lse^2; sums[0..3] += (sum a loss_rows, text-row CE sum,
    image-row CE sum, sum z lse^2)."""
    L.require_device()
    n_tiles, M = part_max.shape
    _chk(sums, F32, "sums")
    if sums.numel() < 4:
        raise L.DB200Error("ce_finish_weighted: sums needs 4 elements")
    ws = L.workspace(L.load().db200_ce_finish_weighted_workspace_bytes(M))
    check(L.load().db200_ce_finish_weighted(stream_ptr(), ptr(part_max), ptr(part_sum), ptr(label_logit), ptr(lse),
                                            ptr(loss_rows), ptr(sums), M, n_tiles, ctypes.byref(weights), ptr(ws),
                                            _nbytes(ws)),
          "db200_ce_finish_weighted")


def logits_mask_partition(hf, labels, bias, hf_text, hf_image, labels_text, labels_image, bias_image, B, S, text_rows,
                          c0, image_offset, V):
    """Row partition of the modality logits mask (include/dalle_b200.h): hf [B*S, d] -> hf_text [B*text_rows, d] and
    hf_image [B*(S - text_rows), d]; labels -> labels_text and labels_image - c0; bias_image [round_up(V - c0, 8)] =
    -inf on [c0, image_offset), bias[image_offset:V], then 0.  With text_rows 0 the text blocks may be None."""
    L.require_device()
    _chk(hf, BF16, "hf"); _chk(hf_text, BF16, "hf_text"); _chk(hf_image, BF16, "hf_image")
    _chk(labels, I32, "labels"); _chk(labels_text, I32, "labels_text"); _chk(labels_image, I32, "labels_image")
    _chk(bias, F32, "bias"); _chk(bias_image, F32, "bias_image")
    d = hf.shape[1]
    ni = S - text_rows
    n_bias = (V - c0 + 7) // 8 * 8
    if tuple(hf.shape) != (B * S, d) or labels.numel() != B * S or tuple(hf_image.shape) != (B * ni, d) or \
            labels_image.numel() != B * ni or bias_image.numel() < n_bias or bias.numel() < V or \
            (text_rows and (tuple(hf_text.shape) != (B * text_rows, d) or labels_text.numel() != B * text_rows)):
        raise L.DB200Error(f"logits_mask_partition: block shapes do not match B={B} S={S} text_rows={text_rows} d={d}")
    check(L.load().db200_logits_mask_partition(stream_ptr(), ptr(hf), ptr(labels), ptr(bias), ptr(hf_text),
                                               ptr(hf_image), ptr(labels_text), ptr(labels_image), ptr(bias_image), B,
                                               S, text_rows, d, int(c0), int(image_offset), int(V)),
          "logits_mask_partition")


def logits_mask_scatter(B, S, text_rows, dx_text=None, dx_image=None, dx=None, loss_text=None, loss_image=None,
                        loss_rows=None):
    """Inverse of logits_mask_partition on row data: dx [B*S, d] from the blocks' dgrads dx_text / dx_image and
    loss_rows [B*S] from loss_text / loss_image (either part skipped when dx, resp. loss_rows, is None)."""
    L.require_device()
    _chk(dx_text, BF16, "dx_text"); _chk(dx_image, BF16, "dx_image"); _chk(dx, BF16, "dx")
    _chk(loss_text, F32, "loss_text"); _chk(loss_image, F32, "loss_image"); _chk(loss_rows, F32, "loss_rows")
    ni = S - text_rows
    d = dx.shape[1] if dx is not None else 0
    if dx is not None and (tuple(dx.shape) != (B * S, d) or tuple(dx_image.shape) != (B * ni, d) or
                           (text_rows and tuple(dx_text.shape) != (B * text_rows, d))):
        raise L.DB200Error(f"logits_mask_scatter: dx block shapes do not match B={B} S={S} text_rows={text_rows}")
    if loss_rows is not None and (loss_rows.numel() != B * S or loss_image.numel() != B * ni or
                                  (text_rows and loss_text.numel() != B * text_rows)):
        raise L.DB200Error(f"logits_mask_scatter: loss block sizes do not match B={B} S={S} text_rows={text_rows}")
    check(L.load().db200_logits_mask_scatter(stream_ptr(), ptr(dx_text), ptr(dx_image), ptr(dx), ptr(loss_text),
                                             ptr(loss_image), ptr(loss_rows), B, S, text_rows, d),
          "logits_mask_scatter")


# ----------------------------------------------------------------------------------------------- row ops
def embed_fwd(ids, wte, wpe, out, wte_drop=None, wpe_drop=None):
    """out = wte[ids] + wpe[s]; with embedding dropout (lib.Dropout descriptors of the wte / wpe sites) each term is
    multiplied by its keep mask * scale."""
    L.require_device()
    _chk(ids, I32, "ids"); _chk(wte, BF16, "wte"); _chk(wpe, BF16, "wpe"); _chk(out, BF16, "out")
    B, S = ids.shape
    V, d = wte.shape
    if wte_drop is None and wpe_drop is None:
        check(L.load().db200_embed_fwd(stream_ptr(), ptr(ids), ptr(wte), ptr(wpe), ptr(out), B, S, d, V), "embed_fwd")
    else:
        check(L.load().db200_embed_fwd_ex(stream_ptr(), ptr(ids), ptr(wte), ptr(wpe), ptr(out), B, S, d, V,
                                          _ref(wte_drop), _ref(wpe_drop)), "embed_fwd_ex")
    return out


def embed_bwd(ids, dx, dwte, dwpe, wte_drop=None, wpe_drop=None, alpha=None):
    """alpha (the stable option's gradient shrink, None: off): every dx element is multiplied by alpha in fp32 before
    it is summed into dwte / dwpe."""
    L.require_device()
    _chk(ids, I32, "ids"); _chk(dx, BF16, "dx"); _chk(dwte, F32, "dwte"); _chk(dwpe, F32, "dwpe")
    B, S = ids.shape
    V, d = dwte.shape
    ws = L.workspace(L.load().db200_embed_bwd_workspace_bytes(d, V))
    if alpha is not None:
        check(L.load().db200_embed_bwd_scaled(stream_ptr(), ptr(ids), ptr(dx), ptr(dwte), ptr(dwpe), B, S, d, V,
                                              ptr(ws), _nbytes(ws), _ref(wte_drop), _ref(wpe_drop), float(alpha)),
              "embed_bwd_scaled")
    elif wte_drop is None and wpe_drop is None:
        check(L.load().db200_embed_bwd(stream_ptr(), ptr(ids), ptr(dx), ptr(dwte), ptr(dwpe), B, S, d, V, ptr(ws),
                                       _nbytes(ws)), "embed_bwd")
    else:
        check(L.load().db200_embed_bwd_ex(stream_ptr(), ptr(ids), ptr(dx), ptr(dwte), ptr(dwpe), B, S, d, V, ptr(ws),
                                          _nbytes(ws), _ref(wte_drop), _ref(wpe_drop)), "embed_bwd_ex")


def assemble_tokens(text_ids, image_idx, tokens, image_offset, caption_drop=None, pad_id=None):
    """tokens = concat(text_ids, image_idx + image_offset) per row.  caption_drop (lib.Dropout of site
    lib.SITE_CAPTION, row0 = global index of row 0): a dropped row's caption is pad_id at every text position."""
    L.require_device()
    _chk(text_ids, I32, "text_ids"); _chk(image_idx, I32, "image_idx"); _chk(tokens, I32, "tokens")
    B, Tt = text_ids.shape
    Ti = image_idx.shape[1]
    if caption_drop is None:
        check(L.load().db200_assemble_tokens(stream_ptr(), ptr(text_ids), ptr(image_idx), ptr(tokens), B, Tt, Ti,
                                             image_offset), "assemble_tokens")
    else:
        check(L.load().db200_assemble_tokens_ex(stream_ptr(), ptr(text_ids), ptr(image_idx), ptr(tokens), B, Tt, Ti,
                                                image_offset, int(pad_id), ctypes.byref(caption_drop)),
              "assemble_tokens_ex")
    return tokens


def assemble_tokens_pp(text_ids, image_idx, tokens, image_offset, pad_id, pad_base, caption_drop=None):
    """assemble_tokens with per-position padding: text position t becomes pad_base + t where the caption id is pad_id
    or the row's caption is dropped (caption_drop as in assemble_tokens).  image_idx None: captions alone (tokens
    [B, text_len])."""
    L.require_device()
    _chk(text_ids, I32, "text_ids"); _chk(image_idx, I32, "image_idx"); _chk(tokens, I32, "tokens")
    B, Tt = text_ids.shape
    Ti = 0 if image_idx is None else image_idx.shape[1]
    if tuple(tokens.shape) != (B, Tt + Ti):
        raise L.DB200Error(f"assemble_tokens_pp: tokens must be [{B}, {Tt + Ti}], got {tuple(tokens.shape)}")
    check(L.load().db200_assemble_tokens_pp(stream_ptr(), ptr(text_ids), ptr(image_idx), ptr(tokens), B, Tt, Ti,
                                            int(image_offset), int(pad_id), int(pad_base), _ref(caption_drop)),
          "assemble_tokens_pp")
    return tokens


def pos_compose(wpe, image_row, image_col, out):
    """out bf16 [TL + W^2, d] = wpe [TL, d] followed by image_row[r] + image_col[c] at TL + r W + c (bf16, each sum
    rounded to nearest even)."""
    L.require_device()
    _chk(wpe, BF16, "wpe"); _chk(image_row, BF16, "image_row"); _chk(image_col, BF16, "image_col"); _chk(out, BF16, "out")
    TL, d = wpe.shape
    W = image_row.shape[0]
    if tuple(image_col.shape) != (W, d) or tuple(image_row.shape) != (W, d) or tuple(out.shape) != (TL + W * W, d):
        raise L.DB200Error(f"pos_compose: shapes wpe {tuple(wpe.shape)} image_row {tuple(image_row.shape)} "
                           f"image_col {tuple(image_col.shape)} out {tuple(out.shape)}")
    check(L.load().db200_pos_compose(stream_ptr(), ptr(wpe), ptr(image_row), ptr(image_col), ptr(out), TL, W, d),
          "pos_compose")
    return out


def pos_fold(dpos, dwpe, dimage_row, dimage_col):
    """dwpe [TL, d] += dpos[:TL]; dimage_row[r] += sum_c dpos[TL + r W + c]; dimage_col[c] += sum_r (fp32, fixed
    order)."""
    L.require_device()
    _chk(dpos, F32, "dpos"); _chk(dwpe, F32, "dwpe"); _chk(dimage_row, F32, "dimage_row")
    _chk(dimage_col, F32, "dimage_col")
    TL, d = dwpe.shape
    W = dimage_row.shape[0]
    if tuple(dimage_col.shape) != (W, d) or tuple(dimage_row.shape) != (W, d) or tuple(dpos.shape) != (TL + W * W, d):
        raise L.DB200Error(f"pos_fold: shapes dpos {tuple(dpos.shape)} dwpe {tuple(dwpe.shape)} dimage_row "
                           f"{tuple(dimage_row.shape)} dimage_col {tuple(dimage_col.shape)}")
    check(L.load().db200_pos_fold(stream_ptr(), ptr(dpos), ptr(dwpe), ptr(dimage_row), ptr(dimage_col), TL, W, d),
          "pos_fold")


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


def layernorm_residual_fwd(o, x_res, g, b, y, mean, rstd, eps=1e-5):
    """Sandwich LayerNorm: y = bf16(x_res + LN(o) * g + b) with LN's statistics of o into mean / rstd (fp32)."""
    L.require_device()
    _chk(o, BF16, "o"); _chk(x_res, BF16, "x_res"); _chk(y, BF16, "y"); _chk(g, F32, "g"); _chk(b, F32, "b")
    _chk(mean, F32, "mean"); _chk(rstd, F32, "rstd")
    rows, d = o.shape
    if tuple(x_res.shape) != (rows, d) or tuple(y.shape) != (rows, d) or mean.numel() < rows or rstd.numel() < rows \
            or g.numel() != d or b.numel() != d:
        raise L.DB200Error(f"layernorm_residual_fwd: o, x_res and y must be [{rows}, {d}], g and b [{d}], mean and "
                           f"rstd >= {rows} entries")
    check(L.load().db200_layernorm_residual_fwd(stream_ptr(), ptr(o), ptr(x_res), ptr(g), ptr(b), ptr(y), ptr(mean),
                                                ptr(rstd), rows, d, eps), "layernorm_residual_fwd")
    return y


def _rows_like(what, rows, d, *tensors):
    for t in tensors:
        if t is not None and (tuple(t.shape) != (rows, d) or not t.is_contiguous()):
            raise L.DB200Error(f"{what}: every [rows, d] operand must be contiguous [{rows}, {d}]")


def layernorm_scale_residual_fwd(o, x_res, g, b, s, y, mean, rstd, eps=1e-5):
    """Sandwich LayerNorm under LayerScale: y = bf16(x_res + s * (LN(o) * g + b)) with LN's statistics of o into mean /
    rstd (fp32), the same values layernorm_fwd writes."""
    L.require_device()
    _chk(o, BF16, "o"); _chk(x_res, BF16, "x_res"); _chk(y, BF16, "y"); _chk(g, F32, "g"); _chk(b, F32, "b")
    _chk(s, F32, "s"); _chk(mean, F32, "mean"); _chk(rstd, F32, "rstd")
    rows, d = o.shape
    _rows_like("layernorm_scale_residual_fwd", rows, d, o, x_res, y)
    if mean.numel() < rows or rstd.numel() < rows or g.numel() != d or b.numel() != d or s.numel() != d:
        raise L.DB200Error(f"layernorm_scale_residual_fwd: g, b and s must have {d} entries, mean and rstd >= {rows}")
    check(L.load().db200_layernorm_scale_residual_fwd(stream_ptr(), ptr(o), ptr(x_res), ptr(g), ptr(b), ptr(s), ptr(y),
                                                      ptr(mean), ptr(rstd), rows, d, eps),
          "layernorm_scale_residual_fwd")
    return y


def layernorm_divmax_fwd(x, g, b, y, mean, rstd, m, eps=1e-5):
    """DivideMax LayerNorm: per row m = max(x) (into m), u = x / m in fp32, y = bf16(LN(u) g + b) with u's statistics
    into mean / rstd."""
    L.require_device()
    _chk(x, BF16, "x"); _chk(y, BF16, "y"); _chk(g, F32, "g"); _chk(b, F32, "b"); _chk(mean, F32, "mean")
    _chk(rstd, F32, "rstd"); _chk(m, F32, "m")
    rows, d = x.shape
    _rows_like("layernorm_divmax_fwd", rows, d, x, y)
    if min(mean.numel(), rstd.numel(), m.numel()) < rows or g.numel() != d or b.numel() != d:
        raise L.DB200Error(f"layernorm_divmax_fwd: g and b must have {d} entries, mean, rstd and m >= {rows}")
    check(L.load().db200_layernorm_divmax_fwd(stream_ptr(), ptr(x), ptr(g), ptr(b), ptr(y), ptr(mean), ptr(rstd),
                                              ptr(m), rows, d, eps), "layernorm_divmax_fwd")
    return y


def layernorm_divmax_bwd(dy, x, g, mean, rstd, m, dres, dx, dg, db, dxsum=None, dxm=None, dropout=None):
    """Backward of layernorm_divmax_fwd with m constant: dx = LN'(x / m)^T dy / m (+ dres); dg, db, and the fusions of
    layernorm_bwd (dxsum; dxm and the dropout site)."""
    L.require_device()
    _chk(dy, BF16, "dy"); _chk(x, BF16, "x"); _chk(dres, BF16, "dres"); _chk(dx, BF16, "dx"); _chk(m, F32, "m")
    _chk(g, F32, "g"); _chk(dg, F32, "dg"); _chk(db, F32, "db"); _chk(dxsum, F32, "dxsum"); _chk(dxm, BF16, "dxm")
    _chk(mean, F32, "mean"); _chk(rstd, F32, "rstd")
    rows, d = x.shape
    _rows_like("layernorm_divmax_bwd", rows, d, dy, x, dres, dx, dxm)
    if min(mean.numel(), rstd.numel(), m.numel()) < rows or g.numel() != d or dg.numel() != d or db.numel() != d \
            or (dxsum is not None and dxsum.numel() != d):
        raise L.DB200Error(f"layernorm_divmax_bwd: mean, rstd and m must have >= {rows} entries, g, dg, db and dxsum "
                           f"{d}")
    ws = L.workspace(L.load().db200_layernorm_bwd_workspace_bytes(rows, d))
    check(L.load().db200_layernorm_divmax_bwd(stream_ptr(), ptr(dy), ptr(x), ptr(g), ptr(mean), ptr(rstd), ptr(m),
                                              ptr(dres), ptr(dx), ptr(dxm), ptr(dg), ptr(db), ptr(dxsum), rows, d,
                                              _ref(dropout), ptr(ws), _nbytes(ws)), "layernorm_divmax_bwd")
    return dx


def layer_scale_residual_fwd(o, x_res, s, y):
    """LayerScale: y = bf16(x_res + s * o), s fp32 [d] per channel."""
    L.require_device()
    _chk(o, BF16, "o"); _chk(x_res, BF16, "x_res"); _chk(y, BF16, "y"); _chk(s, F32, "s")
    rows, d = o.shape
    _rows_like("layer_scale_residual_fwd", rows, d, o, x_res, y)
    if s.numel() != d:
        raise L.DB200Error(f"layer_scale_residual_fwd: s must have {d} entries")
    check(L.load().db200_layer_scale_residual_fwd(stream_ptr(), ptr(o), ptr(x_res), ptr(s), ptr(y), rows, d),
          "layer_scale_residual_fwd")
    return y


def layer_scale_bwd(dy, v, s, dv, ds, db=None, dropout=None, norm=None):
    """LayerScale backward from the residual gradient dy: dv = bf16(s * dy) (times the keep mask and scale of the
    residual-dropout site `dropout`), ds += colsum(dy * v), db (optional) += colsum(dv).  norm = (g, b, mean, rstd):
    v is a sandwich LayerNorm's input o and the scaled value is LN(o) * g + b, recomputed in fp32 (no dropout then)."""
    L.require_device()
    _chk(dy, BF16, "dy"); _chk(v, BF16, "v"); _chk(dv, BF16, "dv"); _chk(s, F32, "s"); _chk(ds, F32, "ds")
    _chk(db, F32, "db")
    rows, d = v.shape
    _rows_like("layer_scale_bwd", rows, d, dy, v, dv)
    g = b = mean = rstd = None
    if norm is not None:
        g, b, mean, rstd = norm
        _chk(g, F32, "g"); _chk(b, F32, "b"); _chk(mean, F32, "mean"); _chk(rstd, F32, "rstd")
        if g.numel() != d or b.numel() != d or mean.numel() < rows or rstd.numel() < rows:
            raise L.DB200Error(f"layer_scale_bwd: g and b must have {d} entries, mean and rstd >= {rows}")
    if s.numel() != d or ds.numel() != d or (db is not None and db.numel() != d):
        raise L.DB200Error(f"layer_scale_bwd: s, ds and db must have {d} entries")
    ws = L.workspace(L.load().db200_layer_scale_bwd_workspace_bytes(rows, d))
    check(L.load().db200_layer_scale_bwd(stream_ptr(), ptr(dy), ptr(v), ptr(s), ptr(g), ptr(b), ptr(mean), ptr(rstd),
                                         ptr(dv), ptr(ds), ptr(db), _ref(dropout), rows, d, ptr(ws), _nbytes(ws)),
          "layer_scale_bwd")
    return dv


def layernorm_bwd(dy, x, g, mean, rstd, dres, dx, dg, db, dxsum=None, dxm=None, dropout=None):
    """dxsum (optional, f32 [d]): += column sums of the produced dx (fused bias gradient of the layer below).
    dxm (with `dropout`, the residual-dropout site of the branch below): also writes dxm = dx * keep * scale, and dxsum
    then sums dxm."""
    L.require_device()
    _chk(dy, BF16, "dy"); _chk(x, BF16, "x"); _chk(dres, BF16, "dres"); _chk(dx, BF16, "dx")
    _chk(g, F32, "g"); _chk(dg, F32, "dg"); _chk(db, F32, "db"); _chk(dxsum, F32, "dxsum"); _chk(dxm, BF16, "dxm")
    rows, d = x.shape
    ws = L.workspace(L.load().db200_layernorm_bwd_workspace_bytes(rows, d))
    if dxm is None:
        check(L.load().db200_layernorm_bwd_ex(stream_ptr(), ptr(dy), ptr(x), ptr(g), ptr(mean), ptr(rstd), ptr(dres),
                                              ptr(dx), ptr(dg), ptr(db), ptr(dxsum), rows, d, ptr(ws), _nbytes(ws)),
              "layernorm_bwd")
    else:
        check(L.load().db200_layernorm_bwd_dropout(stream_ptr(), ptr(dy), ptr(x), ptr(g), ptr(mean), ptr(rstd),
                                                   ptr(dres), ptr(dx), ptr(dxm), ptr(dg), ptr(db), ptr(dxsum), rows, d,
                                                   _ref(dropout), ptr(ws), _nbytes(ws)), "layernorm_bwd_dropout")
    return dx


def dropout_mask(desc, layout, dims, keep):
    """keep (uint8, contiguous): 1 where the site `desc` keeps the element.  layout lib.DROPOUT_ELEMENTWISE with
    dims (rows, cols) -> [rows, cols]; lib.DROPOUT_ATTENTION with dims (B, H, S) -> [B, H, S, S]."""
    L.require_device()
    _chk(keep, torch.uint8, "keep")
    dims = tuple(int(x) for x in dims) + (0,) * (3 - len(dims))
    check(L.load().db200_dropout_mask(stream_ptr(), ctypes.byref(desc), int(layout), dims[0], dims[1], dims[2],
                                      ptr(keep)), "dropout_mask")
    return keep


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
# S x S logits: 4 S^2 dh B H / 2; backward = 2.5 x that (5 products).  A local launch counts the (query, key) pairs of
# its band instead: sum_i min(i + 1, radius); an axial (convolutional, block-sparse) launch those of its mask
# (attn_pairs_axial, attn_pairs_conv, attn_pairs_block_sparse).
ATTN_PROFILE = None


def attn_pairs(S, radius=None):
    """(query, key) pairs a causal (radius None) or local attention of length S computes: sum_i min(i + 1, radius)."""
    if radius is None or radius >= S:
        return S * S / 2.0      # the causal count bench.py has always used (the diagonal counted half)
    r = int(radius)
    return r * (r + 1) / 2.0 + (S - r) * r


def attn_pairs_axial(S, text_len, grid_w, axis):
    """(query, key) pairs an axial attention of length S computes: i + 1 for a text query i, text_len + c + 1 (row,
    axis 0) or text_len + r + 1 (column, axis 1) for the image query at grid row r, column c."""
    m, n = min(S, text_len), max(S - text_len, 0)
    q, rem = divmod(n, grid_w)
    image = q * grid_w * (grid_w + 1) // 2 + rem * (rem + 1) // 2 if axis == 0 else \
        grid_w * q * (q + 1) // 2 + rem * (q + 1)
    return float(m * (m + 1) // 2 + n * text_len + image)


def attn_pairs_conv(S, text_len, grid_w, kernel):
    """(query, key) pairs a convolutional attention of length S computes: i + 1 for a text query i, text_len +
    min(kernel, r + 1) min(kernel, c + 1) for the image query at grid row r, column c."""
    k = kernel

    def run(n):   # sum_{i < n} min(k, i + 1)
        return n * (n + 1) // 2 if n <= k else k * (k + 1) // 2 + (n - k) * k

    m, n = min(S, text_len), max(S - text_len, 0)
    q, rem = divmod(n, grid_w)
    image = run(q) * run(grid_w) + min(k, q + 1) * run(rem)
    return float(m * (m + 1) // 2 + n * text_len + image)


def attn_pairs_block_sparse(S, layout, block):
    """(query, key) pairs a block-sparse attention of length S computes: the pairs j <= i < S with
    layout[i // block][j // block] set."""
    import numpy as np
    lay = np.asarray(layout, dtype=bool)
    n = -(-S // block)
    size = np.minimum(block, S - block * np.arange(n))   # positions of each block below S
    lay = np.tril(lay[:n, :n], -1)
    diag = np.asarray(layout, dtype=bool).diagonal()[:n]
    return float(size @ lay @ size + (diag * size * (size + 1) // 2).sum())


class BlockSparse:
    """The mask of a block-sparse attention layer of length S: layout[r][c] (bool [ceil(S / block)]^2, lower
    triangular) lets the queries of block r see the keys of block c, under the causal mask; block is a multiple of 16.
    Holds it as the kernels read it (include/dalle_b200.h): `tiles`, int16 [ceil(S / 64)]^2 tile masks for
    db200_attn_block_sparse_fwd / _bwd, and `blocks`, int32 [ceil(S / 16), ceil(S / 16) + 1] block lists for
    db200_attn_decode_block_sparse(_dev).  A launch of length P <= S (a prefill) uses the same tables."""

    def __init__(self, layout, block, S, device="cuda"):
        import numpy as np
        lay = np.asarray(layout, dtype=bool)
        nb = -(-S // block)
        if block < 16 or block % 16 or lay.shape != (nb, nb) or (np.triu(lay, 1)).any():
            raise L.DB200Error(f"BlockSparse: a lower-triangular [{nb}, {nb}] layout of blocks of a multiple of 16 "
                               f"tokens is needed for S {S}, got shape {lay.shape}, block {block}")
        self.layout, self.block, self.S = lay, int(block), int(S)
        f = block // 16
        ng = -(-S // 16)
        g = np.arange(ng) // f
        lay16 = np.tril(lay[g][:, g])             # the layout at 16-token granularity, [ng, ng]
        nt = -(-S // 64)
        pad = np.zeros((4 * nt, 4 * nt), dtype=bool)
        pad[:ng, :ng] = lay16
        bits = pad.reshape(nt, 4, nt, 4).transpose(0, 2, 1, 3).reshape(nt, nt, 16)   # [qt, kt, 4 a + c]
        tiles = (bits.astype(np.int64) << np.arange(16)).sum(-1)
        self.tiles = torch.from_numpy(tiles.astype(np.uint16).view(np.int16)).to(device)
        lists = np.zeros((ng, ng + 1), dtype=np.int32)
        for r in range(ng):
            cols = np.flatnonzero(lay16[r])
            lists[r, 0] = cols.size
            lists[r, 1:1 + cols.size] = cols
        self.blocks = torch.from_numpy(lists).to(device)

    def pairs(self, S):
        return attn_pairs_block_sparse(S, self.layout, self.block)


def _attn_timed(kind, B, S, H, dh, call, radius=None, axial=None, conv=None, block_sparse=None):
    prof = ATTN_PROFILE
    if prof is None:
        return call()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    call()
    ev1.record()
    pairs = attn_pairs_axial(S, *axial) if axial is not None else \
        attn_pairs_conv(S, *conv) if conv is not None else \
        block_sparse.pairs(S) if block_sparse is not None else attn_pairs(S, radius)
    prof.append((ev0, ev1, 4.0 * pairs * dh * B * H * (1.0 if kind == "fwd" else 2.5), kind))


def _radius(radius):
    if radius is None:
        return None
    if isinstance(radius, bool) or int(radius) != radius or radius < 1:
        raise L.DB200Error(f"attention radius must be an integer >= 1 (or None), got {radius!r}")
    return int(radius)


def _axial(axial, radius, dropout, what):
    """Validated (text_len, grid_w, axis) of an axial launch, or None."""
    if axial is None:
        return None
    if radius is not None or dropout is not None:
        raise L.DB200Error(f"{what}: axial attention takes no radius and no dropout")
    if len(axial) != 3 or any(not isinstance(v, numbers.Integral) or isinstance(v, bool) for v in axial):
        raise L.DB200Error(f"{what}: axial must be three integers (text_len, grid_w, axis), got {axial!r}")
    return tuple(int(v) for v in axial)


def _conv(conv, radius, axial, dropout, what):
    """Validated (text_len, grid_w, kernel) of a convolutional launch, or None."""
    if conv is None:
        return None
    if radius is not None or axial is not None or dropout is not None:
        raise L.DB200Error(f"{what}: convolutional attention takes no radius, no axial geometry and no dropout")
    if len(conv) != 3 or any(not isinstance(v, numbers.Integral) or isinstance(v, bool) for v in conv):
        raise L.DB200Error(f"{what}: conv must be three integers (text_len, grid_w, kernel), got {conv!r}")
    return tuple(int(v) for v in conv)


def _block_sparse(bs, radius, axial, conv, dropout, S, what):
    """Validated BlockSparse of a block-sparse launch of length S, or None."""
    if bs is None:
        return None
    if radius is not None or axial is not None or conv is not None or dropout is not None:
        raise L.DB200Error(f"{what}: block-sparse attention takes no radius, no axial or conv geometry and no dropout")
    if not isinstance(bs, BlockSparse):
        raise L.DB200Error(f"{what}: block_sparse must be an ops.BlockSparse, got {type(bs).__name__}")
    if S > bs.S:
        raise L.DB200Error(f"{what}: length {S} exceeds the block-sparse layout's {bs.S}")
    return bs


def attn_fwd(qkv, out, lse, B, S, H, dh, scale=1.0, dropout=None, radius=None, axial=None, conv=None,
             block_sparse=None):
    """dropout: lib.Dropout of the attention-weights site (row0 = global index of sequence 0), or None.
    radius: None = causal attention; else local attention, query i over keys (i - radius, i] (no dropout).
    axial: (text_len, grid_w, axis) = row (axis 0) or column (axis 1) attention of the image tokens of a text_len
    caption and a grid_w x grid_w image (db200_attn_axial_fwd); excludes radius and dropout.
    conv: (text_len, grid_w, kernel) = convolutional attention over the same grid, the image query at (r, c) over the
    caption and the kernel x kernel window of image tokens (r - kernel, r] x (c - kernel, c] (db200_attn_conv_fwd);
    excludes radius, axial and dropout.
    block_sparse: a BlockSparse of length >= S = block-sparse attention over its layout (db200_attn_block_sparse_fwd);
    excludes radius, axial, conv and dropout."""
    L.require_device()
    _chk(qkv, BF16, "qkv"); _chk(out, BF16, "out"); _chk(lse, F32, "lse")
    bs = _block_sparse(block_sparse, radius, axial, conv, dropout, S, "attn_fwd")
    conv = _conv(conv, radius, axial, dropout, "attn_fwd")
    axial = _axial(axial, radius, dropout, "attn_fwd")
    radius = _radius(radius)
    if bs is not None:
        call = lambda: check(L.load().db200_attn_block_sparse_fwd(stream_ptr(), ptr(qkv), ptr(out), ptr(lse), B, S, H,
                                                                  dh, ptr(bs.tiles), bs.tiles.shape[1], scale),
                             "attn_block_sparse_fwd")
    elif conv is not None:
        call = lambda: check(L.load().db200_attn_conv_fwd(stream_ptr(), ptr(qkv), ptr(out), ptr(lse), B, S, H, dh,
                                                          *conv, scale), "attn_conv_fwd")
    elif axial is not None:
        call = lambda: check(L.load().db200_attn_axial_fwd(stream_ptr(), ptr(qkv), ptr(out), ptr(lse), B, S, H, dh,
                                                           *axial, scale), "attn_axial_fwd")
    elif radius is not None:
        if dropout is not None:
            raise L.DB200Error("attn_fwd: local attention has no dropout (src/dalle_mtf/models.py:270)")
        call = lambda: check(L.load().db200_attn_local_fwd(stream_ptr(), ptr(qkv), ptr(out), ptr(lse), B, S, H, dh,
                                                           radius, scale), "attn_local_fwd")
    elif dropout is None:
        call = lambda: check(L.load().db200_attn_causal_fwd(stream_ptr(), ptr(qkv), ptr(out), ptr(lse), B, S, H, dh,
                                                            scale), "attn_causal_fwd")
    else:
        call = lambda: check(L.load().db200_attn_causal_fwd_ex(stream_ptr(), ptr(qkv), ptr(out), ptr(lse), B, S, H, dh,
                                                               scale, ctypes.byref(dropout)), "attn_causal_fwd_ex")
    _attn_timed("fwd", B, S, H, dh, call, radius, axial, conv, bs)
    return out


def attn_bwd(qkv, out, dout, lse, dq_accum, delta, dqkv, B, S, H, dh, scale=1.0, dropout=None, radius=None,
             axial=None, conv=None, block_sparse=None):
    """radius, axial, conv, block_sparse: as attn_fwd's (None = causal)."""
    L.require_device()
    _chk(qkv, BF16, "qkv"); _chk(out, BF16, "out"); _chk(dout, BF16, "dout"); _chk(dqkv, BF16, "dqkv")
    _chk(lse, F32, "lse"); _chk(dq_accum, F32, "dq_accum"); _chk(delta, F32, "delta")
    bs = _block_sparse(block_sparse, radius, axial, conv, dropout, S, "attn_bwd")
    conv = _conv(conv, radius, axial, dropout, "attn_bwd")
    axial = _axial(axial, radius, dropout, "attn_bwd")
    radius = _radius(radius)
    if bs is not None:
        call = lambda: check(L.load().db200_attn_block_sparse_bwd(stream_ptr(), ptr(qkv), ptr(out), ptr(dout), ptr(lse),
                                                                  ptr(dq_accum), ptr(delta), ptr(dqkv), B, S, H, dh,
                                                                  ptr(bs.tiles), bs.tiles.shape[1], scale),
                             "attn_block_sparse_bwd")
    elif conv is not None:
        call = lambda: check(L.load().db200_attn_conv_bwd(stream_ptr(), ptr(qkv), ptr(out), ptr(dout), ptr(lse),
                                                          ptr(dq_accum), ptr(delta), ptr(dqkv), B, S, H, dh, *conv,
                                                          scale), "attn_conv_bwd")
    elif axial is not None:
        call = lambda: check(L.load().db200_attn_axial_bwd(stream_ptr(), ptr(qkv), ptr(out), ptr(dout), ptr(lse),
                                                           ptr(dq_accum), ptr(delta), ptr(dqkv), B, S, H, dh, *axial,
                                                           scale), "attn_axial_bwd")
    elif radius is not None:
        if dropout is not None:
            raise L.DB200Error("attn_bwd: local attention has no dropout (src/dalle_mtf/models.py:270)")
        call = lambda: check(L.load().db200_attn_local_bwd(stream_ptr(), ptr(qkv), ptr(out), ptr(dout), ptr(lse),
                                                           ptr(dq_accum), ptr(delta), ptr(dqkv), B, S, H, dh, radius,
                                                           scale), "attn_local_bwd")
    elif dropout is None:
        call = lambda: check(L.load().db200_attn_causal_bwd(stream_ptr(), ptr(qkv), ptr(out), ptr(dout), ptr(lse),
                                                            ptr(dq_accum), ptr(delta), ptr(dqkv), B, S, H, dh, scale),
                             "attn_causal_bwd")
    else:
        call = lambda: check(L.load().db200_attn_causal_bwd_ex(stream_ptr(), ptr(qkv), ptr(out), ptr(dout), ptr(lse),
                                                               ptr(dq_accum), ptr(delta), ptr(dqkv), B, S, H, dh,
                                                               scale, ctypes.byref(dropout)), "attn_causal_bwd_ex")
    _attn_timed("bwd", B, S, H, dh, call, radius, axial, conv, bs)
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


# the DALL-E paper's dVAE network (include/dalle_b200.h, K11p): activations NHWC, bf16 or f32 (all operands alike)
def _act(t, name, *others):
    """act_f32 flag of activation tensor t; every tensor in `others` must have its dtype."""
    if t.dtype not in (BF16, F32):
        raise L.DB200Error(f"{name}: activations must be bf16 or f32, got {t.dtype}")
    for o in others:
        _chk(o, t.dtype, name)
    _chk(t, t.dtype, name)
    return int(t.dtype == F32)


def conv7x7_in_fwd(x_f32, w, bias, y):
    """Encoder input conv: f32 image [N,H,W,C] (C <= 4) -> y [N,H,W,Cout] (bf16 or f32) = conv7x7(x, w) + bias
    (SAME, stride 1), f32 FMAs of the f32 operands, the output rounded once."""
    L.require_device()
    _chk(x_f32, F32, "x"); _chk(w, F32, "w"); _chk(bias, F32, "bias")
    N, H, W_, C = x_f32.shape
    if tuple(w.shape) != (7, 7, C, y.shape[-1]) or tuple(y.shape[:3]) != (N, H, W_):
        raise L.DB200Error(f"conv7x7_in_fwd: shapes x {tuple(x_f32.shape)} w {tuple(w.shape)} y {tuple(y.shape)}")
    check(L.load().db200_conv7x7_in_fwd(stream_ptr(), ptr(x_f32), ptr(w), ptr(bias), ptr(y), N, H, W_, C,
                                        y.shape[-1], _act(y, "y")), "conv7x7_in_fwd")
    return y


def conv7x7_in_wgrad(x_f32, dy, dw, dbias):
    """dw [7,7,C,Cout] += the 7x7 input conv's kernel gradient, dbias [Cout] += sum dy (dbias may be None)."""
    L.require_device()
    _chk(x_f32, F32, "x"); _chk(dw, F32, "dw"); _chk(dbias, F32, "dbias")
    N, H, W_, C = x_f32.shape
    Cout = dy.shape[-1]
    if tuple(dw.shape) != (7, 7, C, Cout) or tuple(dy.shape[:3]) != (N, H, W_):
        raise L.DB200Error(f"conv7x7_in_wgrad: shapes x {tuple(x_f32.shape)} dy {tuple(dy.shape)} dw {tuple(dw.shape)}")
    ws = L.workspace(L.load().db200_conv7x7_in_wgrad_workspace_bytes(N, H, W_, C, Cout))
    check(L.load().db200_conv7x7_in_wgrad(stream_ptr(), ptr(x_f32), ptr(dy), ptr(dw), ptr(dbias), N, H, W_, C, Cout,
                                          _act(dy, "dy"), ptr(ws), _nbytes(ws)), "conv7x7_in_wgrad")


def maxpool2x2_fwd(x, y):
    """y [N,H/2,W/2,C] = 2x2 stride-2 max-pool of x [N,H,W,C]."""
    L.require_device()
    N, H, W_, C = x.shape
    check(L.load().db200_maxpool2x2_fwd(stream_ptr(), ptr(x), ptr(y), N, H, W_, C, _act(x, "maxpool2x2_fwd", y)),
          "maxpool2x2_fwd")
    return y


def maxpool2x2_bwd(x, dy, dx):
    """dx [N,H,W,C] = dy at each window's first maximum of x (raster order), 0 elsewhere."""
    L.require_device()
    N, H, W_, C = x.shape
    check(L.load().db200_maxpool2x2_bwd(stream_ptr(), ptr(x), ptr(dy), ptr(dx), N, H, W_, C,
                                        _act(x, "maxpool2x2_bwd", dy, dx)), "maxpool2x2_bwd")
    return dx


def upsample2x_fwd(x, y):
    """y [N,2H,2W,C] = nearest-neighbour 2x upsampling of x [N,H,W,C]."""
    L.require_device()
    N, H, W_, C = x.shape
    check(L.load().db200_upsample2x_fwd(stream_ptr(), ptr(x), ptr(y), N, H, W_, C, _act(x, "upsample2x_fwd", y)),
          "upsample2x_fwd")
    return y


def upsample2x_bwd(dy, dx):
    """dx [N,H,W,C] = the f32 sum of each 2x2 block of dy [N,2H,2W,C]."""
    L.require_device()
    N, H, W_, C = dx.shape
    check(L.load().db200_upsample2x_bwd(stream_ptr(), ptr(dy), ptr(dx), N, H, W_, C, _act(dx, "upsample2x_bwd", dy)),
          "upsample2x_bwd")
    return dx


def residual_gain(r, gain=1.0, id=None, mask=None, y=None, relu_y=None):
    """v = gain * r + id (id None: gain * r), 0 where mask <= 0; y = v (activation dtype), relu_y = max(y, 0)."""
    L.require_device()
    act = _act(r, "residual_gain", id, mask, y, relu_y)
    check(L.load().db200_residual_gain(stream_ptr(), ptr(id), ptr(r), ptr(mask), float(gain), ptr(y), ptr(relu_y),
                                       r.numel(), act), "residual_gain")
    return y if y is not None else relu_y


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


# the VQGAN tokenizer (include/dalle_b200.h, K14): NHWC bf16 activations
def groupnorm_stats(x, mean, rstd, groups=32, eps=1e-6):
    """mean / rstd f32 [N, groups] of x bf16 [N, H, W, C] (biased variance, fp32, fixed-order reduction)."""
    L.require_device()
    _chk(x, BF16, "x"); _chk(mean, F32, "mean"); _chk(rstd, F32, "rstd")
    N, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (N * C)
    if mean.numel() != N * groups or rstd.numel() != N * groups:
        raise L.DB200Error(f"groupnorm_stats: mean / rstd need {N * groups} elements")
    ws = L.workspace(L.load().db200_groupnorm_stats_workspace_bytes(N, HW, C, groups))
    check(L.load().db200_groupnorm_stats(stream_ptr(), ptr(x), ptr(mean), ptr(rstd), N, HW, C, groups, float(eps),
                                         ptr(ws), _nbytes(ws)), "groupnorm_stats")


def groupnorm_apply(x, mean, rstd, gamma, beta, y, groups=32, swish=False):
    """y = (x - mean) rstd gamma + beta [swish], bf16 [N, H, W, C] like x."""
    L.require_device()
    _chk(x, BF16, "x"); _chk(y, BF16, "y"); _chk(gamma, F32, "gamma"); _chk(beta, F32, "beta")
    N, C = x.shape[0], x.shape[-1]
    if tuple(y.shape) != tuple(x.shape) or gamma.numel() != C or beta.numel() != C:
        raise L.DB200Error(f"groupnorm_apply: shapes x {tuple(x.shape)} y {tuple(y.shape)} gamma {tuple(gamma.shape)}")
    check(L.load().db200_groupnorm_apply(stream_ptr(), ptr(x), ptr(mean), ptr(rstd), ptr(gamma), ptr(beta), ptr(y), N,
                                         x.numel() // (N * C), C, groups, int(bool(swish))), "groupnorm_apply")
    return y


def groupnorm(x, mean, rstd, gamma, beta, y, groups=32, eps=1e-6, swish=False):
    groupnorm_stats(x, mean, rstd, groups, eps)
    return groupnorm_apply(x, mean, rstd, gamma, beta, y, groups, swish)


def attn_noncausal(qkv, out, B, S, C, scale):
    """out bf16 [B, S, C] = softmax(scale q k^T) v of each image's q | k | v bf16 [B, S, 3C]."""
    L.require_device()
    _chk(qkv, BF16, "qkv"); _chk(out, BF16, "out")
    if qkv.numel() != B * S * 3 * C or out.numel() != B * S * C:
        raise L.DB200Error(f"attn_noncausal: qkv {tuple(qkv.shape)} / out {tuple(out.shape)} do not match B={B}, "
                           f"S={S}, C={C}")
    check(L.load().db200_attn_noncausal_fwd(stream_ptr(), ptr(qkv), ptr(out), B, S, C, float(scale)),
          "attn_noncausal_fwd")
    return out


def attn_noncausal_long(qkv, out, B, S, C, scale):
    """attn_noncausal over longer sequences on wgmma: C == 512, S % 64 == 0 and 256 < S <= 4096."""
    L.require_device()
    _chk(qkv, BF16, "qkv"); _chk(out, BF16, "out")
    if qkv.numel() != B * S * 3 * C or out.numel() != B * S * C:
        raise L.DB200Error(f"attn_noncausal_long: qkv {tuple(qkv.shape)} / out {tuple(out.shape)} do not match B={B}, "
                           f"S={S}, C={C}")
    check(L.load().db200_attn_noncausal_long_fwd(stream_ptr(), ptr(qkv), ptr(out), B, S, C, float(scale)),
          "attn_noncausal_long_fwd")
    return out


def gather_rows_split(idx, table, hi, lo=None, offset=0):
    """hi [rows, D] = bf16(table[idx - offset]), lo = bf16(row - hi); ids outside [offset, offset + K) give zeros."""
    L.require_device()
    _chk(idx, I32, "idx"); _chk(table, F32, "table"); _chk(hi, BF16, "hi"); _chk(lo, BF16, "lo")
    K, D = table.shape
    rows = idx.numel()
    if hi.numel() != rows * D or (lo is not None and lo.numel() != rows * D):
        raise L.DB200Error(f"gather_rows_split: hi / lo need {rows} x {D} elements")
    check(L.load().db200_gather_rows_split(stream_ptr(), ptr(idx), ptr(table), ptr(hi), ptr(lo), rows, D, K,
                                           int(offset)), "gather_rows_split")


def clamp_bf16_to_f32(src, dst, lo=-1.0, hi=1.0):
    """dst f32 = clamp(src bf16, lo, hi), elementwise."""
    L.require_device()
    _chk(src, BF16, "src"); _chk(dst, F32, "dst")
    if src.numel() != dst.numel():
        raise L.DB200Error("clamp_bf16_to_f32: src and dst sizes differ")
    check(L.load().db200_clamp_bf16_to_f32(stream_ptr(), ptr(src), ptr(dst), src.numel(), float(lo), float(hi)),
          "clamp_bf16_to_f32")
    return dst


def vae_kl_stats(logits, lse, ent, hist, kl_accum, rows, K, scale):
    """KL(softmax(l) || Uniform(K)) statistics of f32 logits [rows, K]: lse / ent f32 [rows] (logsumexp, sum q (l - lse)),
    hist int32 [K] += the first-maximum code counts, kl_accum[0] += scale * sum of the rows' KL."""
    L.require_device()
    _chk(logits, F32, "logits"); _chk(lse, F32, "lse"); _chk(ent, F32, "ent"); _chk(hist, I32, "hist")
    _chk(kl_accum, F32, "kl_accum")
    if logits.numel() < rows * K or lse.numel() < rows or ent.numel() < rows or hist.numel() < K:
        raise L.DB200Error("vae_kl_stats: a buffer is smaller than rows x K")
    ws = L.workspace(L.load().db200_vae_kl_stats_workspace_bytes(rows, K))
    check(L.load().db200_vae_kl_stats(stream_ptr(), ptr(logits), ptr(lse), ptr(ent), ptr(hist), ptr(kl_accum), rows,
                                      K, scale, ptr(ws), _nbytes(ws)), "db200_vae_kl_stats")


def gumbel_softmax_bwd_kl(y_soft, dy, logits, lse, ent, dlogits, rows, K, tau, c):
    """gumbel_softmax_bwd plus the gradient of c * KL: dlogits += c q (l - lse - ent), in the same pass."""
    L.require_device()
    check(L.load().db200_gumbel_softmax_bwd_kl(stream_ptr(), ptr(y_soft), ptr(dy), ptr(logits), ptr(lse), ptr(ent),
                                               ptr(dlogits), rows, K, tau, c), "gumbel_softmax_bwd_kl")


def mse_fwd_bwd(pred, target, dpred, loss_accum, scale):
    L.require_device()
    check(L.load().db200_mse_fwd_bwd(stream_ptr(), ptr(pred), ptr(target), ptr(dpred), ptr(loss_accum),
                                     pred.numel(), scale), "mse_fwd_bwd")


def logit_laplace(stats, target, dstats, recon, nll_accum, mse_accum, n_pix, Cp, scale):
    """Logit-Laplace loss of f32 decoder stats [n_pix, 2 Cp] (mu | ln b) against the packed f32 target [n_pix, Cp] in
    [-1, 1]: recon [n_pix, Cp] = the image-space output, nll_accum[0] / mse_accum[0] += scale * the sums of the NLL and
    of (recon - target)^2, dstats = scale * d(NLL) / d(stats).  target None (decoding): recon only."""
    L.require_device()
    _chk(stats, F32, "stats"); _chk(target, F32, "target"); _chk(dstats, F32, "dstats"); _chk(recon, F32, "recon")
    _chk(nll_accum, F32, "nll_accum"); _chk(mse_accum, F32, "mse_accum")
    if stats.numel() < n_pix * 2 * Cp or recon.numel() < n_pix * Cp or (
            target is not None and (target.numel() < n_pix * Cp or dstats is None or dstats.numel() < n_pix * 2 * Cp)):
        raise L.DB200Error("logit_laplace: a buffer is smaller than n_pix x Cp")
    ws = None if target is None else L.workspace(L.load().db200_logit_laplace_workspace_bytes(n_pix, Cp))
    check(L.load().db200_logit_laplace_fwd_bwd(stream_ptr(), ptr(stats), ptr(target), ptr(dstats), ptr(recon),
                                               ptr(nll_accum), ptr(mse_accum), n_pix, Cp, scale, ptr(ws),
                                               _nbytes(ws)), "db200_logit_laplace_fwd_bwd")


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


def attn_decode(qkv_step, k_cache, v_cache, out, pos, scale, radius=None, axial=None, conv=None, block_sparse=None):
    """Append this position's k, v to the caches and attend with its q over keys <= pos (models.py:246-254, 281-299);
    radius (local layer, models.py:257-273): over keys [max(0, pos - radius + 1), pos] only; axial (text_len, grid_w,
    axis) (row / column layer, attn_fwd's): over the text keys and pos's image row (axis 0) or column (axis 1); conv
    (text_len, grid_w, kernel) (convolutional layer, attn_fwd's): over the text keys and pos's kernel x kernel window;
    block_sparse (a BlockSparse of the caches' length, attn_fwd's): over the keys <= pos of the blocks its layout lets
    pos's block see."""
    L.require_device()
    _chk(qkv_step, BF16, "qkv_step"); _chk(k_cache, BF16, "k_cache"); _chk(v_cache, BF16, "v_cache"); _chk(out, BF16, "out")
    B, S, H, dh = k_cache.shape
    assert v_cache.shape == k_cache.shape and qkv_step.numel() == B * 3 * H * dh and out.numel() == B * H * dh
    bs = _block_sparse(block_sparse, radius, axial, conv, None, S, "attn_decode")
    conv = _conv(conv, radius, axial, None, "attn_decode")
    axial = _axial(axial, radius, None, "attn_decode")
    radius = _radius(radius)
    if bs is not None:
        check(L.load().db200_attn_decode_block_sparse(stream_ptr(), ptr(qkv_step), ptr(k_cache), ptr(v_cache),
                                                      ptr(out), B, S, H, dh, int(pos), ptr(bs.blocks),
                                                      bs.blocks.shape[1], float(scale)),
              "db200_attn_decode_block_sparse")
        return out
    if conv is not None:
        check(L.load().db200_attn_decode_conv(stream_ptr(), ptr(qkv_step), ptr(k_cache), ptr(v_cache), ptr(out), B, S,
                                              H, dh, int(pos), *conv, float(scale)), "db200_attn_decode_conv")
        return out
    if axial is not None:
        check(L.load().db200_attn_decode_axial(stream_ptr(), ptr(qkv_step), ptr(k_cache), ptr(v_cache), ptr(out), B, S,
                                               H, dh, int(pos), *axial, float(scale)), "db200_attn_decode_axial")
        return out
    if radius is not None:
        check(L.load().db200_attn_decode_local(stream_ptr(), ptr(qkv_step), ptr(k_cache), ptr(v_cache), ptr(out), B, S,
                                               H, dh, int(pos), radius, float(scale)), "db200_attn_decode_local")
        return out
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


def attn_decode_dev(qkv_step, k_cache, v_cache, out, pos_dev, scale, radius=None, axial=None, conv=None,
                    block_sparse=None):
    """attn_decode with the position read on the device from pos_dev (graph replay)."""
    L.require_device()
    B, S, H, dh = k_cache.shape
    bs = _block_sparse(block_sparse, radius, axial, conv, None, S, "attn_decode_dev")
    conv = _conv(conv, radius, axial, None, "attn_decode_dev")
    axial = _axial(axial, radius, None, "attn_decode_dev")
    radius = _radius(radius)
    if bs is not None:
        check(L.load().db200_attn_decode_block_sparse_dev(stream_ptr(), ptr(qkv_step), ptr(k_cache), ptr(v_cache),
                                                          ptr(out), B, S, H, dh, ptr(pos_dev), ptr(bs.blocks),
                                                          bs.blocks.shape[1], float(scale)),
              "db200_attn_decode_block_sparse_dev")
        return out
    if conv is not None:
        check(L.load().db200_attn_decode_conv_dev(stream_ptr(), ptr(qkv_step), ptr(k_cache), ptr(v_cache), ptr(out), B,
                                                  S, H, dh, ptr(pos_dev), *conv, float(scale)),
              "db200_attn_decode_conv_dev")
        return out
    if axial is not None:
        check(L.load().db200_attn_decode_axial_dev(stream_ptr(), ptr(qkv_step), ptr(k_cache), ptr(v_cache), ptr(out), B,
                                                   S, H, dh, ptr(pos_dev), *axial, float(scale)),
              "db200_attn_decode_axial_dev")
        return out
    if radius is not None:
        check(L.load().db200_attn_decode_local_dev(stream_ptr(), ptr(qkv_step), ptr(k_cache), ptr(v_cache), ptr(out), B,
                                                   S, H, dh, ptr(pos_dev), radius, float(scale)),
              "db200_attn_decode_local_dev")
        return out
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


def sample_rows_filtered(logits, u, idx, lo, hi, inv_temp, top_k, top_p, kept=None):
    """sample_rows restricted to the top-k / nucleus set of logits * inv_temp over [lo, hi) (top_k 0 and top_p 1 are
    off; ties at either threshold are kept).  kept (int32 [rows], optional) receives the size of each row's kept set."""
    L.require_device()
    _chk(logits, F32, "logits"); _chk(u, F32, "u"); _chk(idx, I32, "idx"); _chk(kept, I32, "kept")
    rows = logits.shape[0]
    if u is not None:
        assert u.shape == (rows, hi - lo)
    check(L.load().db200_sample_rows_filtered(stream_ptr(), ptr(logits), ptr(u), ptr(idx), ptr(kept), rows,
                                              logits.stride(0), int(lo), int(hi), float(inv_temp), int(top_k),
                                              float(top_p)), "db200_sample_rows_filtered")
    return idx


def sample_rows_filtered_at(logits, u, tokens, lo, hi, inv_temp, top_k, top_p, pos_dev, kept=None):
    """tokens[r, pos + 1] = sample_rows_filtered's id for row r   (pos read on the device)."""
    L.require_device()
    _chk(logits, F32, "logits"); _chk(u, F32, "u"); _chk(tokens, I32, "tokens"); _chk(kept, I32, "kept")
    check(L.load().db200_sample_rows_filtered_at(stream_ptr(), ptr(logits), ptr(u), ptr(tokens), tokens.stride(0),
                                                 ptr(kept), logits.shape[0], logits.stride(0), int(lo), int(hi),
                                                 float(inv_temp), int(top_k), float(top_p), ptr(pos_dev)),
          "db200_sample_rows_filtered_at")
    return tokens


def sample_rows_guided(logits, u, tokens, lo, hi, inv_temp, guidance_scale, top_k=0, top_p=1.0, pos_dev=None,
                       kept=None):
    """Classifier-free guidance over R = logits.shape[0] // 2 pairs: logits rows [0, R) conditional, [R, 2R)
    unconditional; pair r draws from u + s (c - u) (rounded op by op) * inv_temp, filtered like sample_rows_filtered
    (top_k 0 and top_p 1 are off: the unfiltered kernel runs).  The id goes to tokens[r, col] and tokens[R + r, col],
    col = pos + 1 with pos read from pos_dev, else 0 (pass e.g. out[:, j:j + 1] to write column j).  u: [R, hi - lo]."""
    L.require_device()
    _chk(logits, F32, "logits"); _chk(u, F32, "u"); _chk(tokens, I32, "tokens"); _chk(kept, I32, "kept")
    _chk(pos_dev, I32, "pos_dev")
    rows2 = logits.shape[0]
    if rows2 % 2 or tokens.shape[0] != rows2:
        raise L.DB200Error(f"sample_rows_guided: logits rows {rows2} must be even and match tokens rows "
                           f"{tokens.shape[0]}")
    rows = rows2 // 2
    if u is not None:
        assert u.shape == (rows, hi - lo)
    check(L.load().db200_sample_rows_guided(stream_ptr(), ptr(logits), logits.stride(0), ptr(u), ptr(tokens),
                                            tokens.stride(0), ptr(kept), rows, int(lo), int(hi), float(inv_temp),
                                            float(guidance_scale), int(top_k), float(top_p), ptr(pos_dev)),
          "db200_sample_rows_guided")
    return tokens


def _caption_args(tokens, prefix, lens, text_len):
    L.require_device()
    _chk(tokens, I32, "tokens"); _chk(prefix, I32, "prefix"); _chk(lens, I32, "lens")
    rows = tokens.shape[0]
    if tokens.dim() != 2 or tokens.stride(1) != 1 or prefix.dim() != 2 or prefix.stride(1) != 1 or \
            prefix.shape[0] != rows or not lens.is_contiguous() or lens.numel() != rows or \
            min(tokens.shape[1], prefix.shape[1]) < text_len:
        raise L.DB200Error(f"caption_next: tokens and prefix must be [{rows}, >= {text_len}] with unit column stride, "
                           f"lens [{rows}]")
    return rows


def caption_next(tokens, prefix, lens, pos, text_len, text_vocab_size, padding_id, pad_base=None):
    """Finish text column c = pos + 1 of the token matrix tokens int32 [rows, >= text_len] after a draw: prefix[b, c]
    (int32, token form) where c < lens[b], else c's pad (pad_base + c with per-position padding, else padding_id) when
    column c - 1 or the draw is a padding token (padding_id, or with pad_base any id >= text_vocab_size)."""
    rows = _caption_args(tokens, prefix, lens, text_len)
    check(L.load().db200_caption_next(stream_ptr(), ptr(tokens), tokens.stride(0), ptr(prefix), prefix.stride(0),
                                      ptr(lens), rows, int(text_len), int(text_vocab_size), int(padding_id),
                                      -1 if pad_base is None else int(pad_base), int(pos)), "db200_caption_next")
    return tokens


def caption_next_at(tokens, prefix, lens, pos_dev, text_len, text_vocab_size, padding_id, pad_base=None):
    """caption_next with the position read on the device from pos_dev (graph replay)."""
    rows = _caption_args(tokens, prefix, lens, text_len)
    _chk(pos_dev, I32, "pos_dev")
    check(L.load().db200_caption_next_at(stream_ptr(), ptr(tokens), tokens.stride(0), ptr(prefix), prefix.stride(0),
                                         ptr(lens), rows, int(text_len), int(text_vocab_size), int(padding_id),
                                         -1 if pad_base is None else int(pad_base), ptr(pos_dev)),
          "db200_caption_next_at")
    return tokens


def kv_cache_fill(qkv, k_cache, v_cache, P, rep=1):
    """k_cache[b*rep + r, p] = qkv[b, p, 1], v_cache[b*rep + r, p] = qkv[b, p, 2] for p < P (qkv [B*P, 3*H*dh], caches
    [B*rep, S_cache, H, dh]); later positions are left as they are."""
    L.require_device()
    _chk(qkv, BF16, "qkv"); _chk(k_cache, BF16, "k_cache"); _chk(v_cache, BF16, "v_cache")
    Brep, S_cache, H, dh = k_cache.shape
    assert v_cache.shape == k_cache.shape and k_cache.is_contiguous() and v_cache.is_contiguous()
    B = Brep // max(int(rep), 1)
    assert qkv.is_contiguous() and qkv.numel() == B * P * 3 * H * dh, "qkv must be [B*P, 3*H*dh]"
    check(L.load().db200_kv_cache_fill(stream_ptr(), ptr(qkv), ptr(k_cache), ptr(v_cache), B, int(P), H, dh, S_cache,
                                       int(rep)), "db200_kv_cache_fill")


def _rope_args(qkv, table, H, dh, r, what):
    """(rows, table positions) of a rotary call after the dtype / shape checks."""
    L.require_device()
    _chk(qkv, BF16, what); _chk(table, F32, "table")
    if not qkv.is_contiguous() or qkv.dim() != 2 or qkv.shape[1] != 3 * H * dh:
        raise L.DB200Error(f"{what}: expected a contiguous [rows, {3 * H * dh}] q|k|v buffer, got {tuple(qkv.shape)}")
    if not table.is_contiguous() or table.dim() != 3 or tuple(table.shape[1:]) != (2, r // 2):
        raise L.DB200Error(f"{what}: expected a contiguous [n_pos, 2, {r // 2}] table, got {tuple(table.shape)}")
    return qkv.shape[0], table.shape[0]


def rope_fwd(qkv, table, S, H, dh, r):
    """Rotary position embedding in place on the q and k columns of qkv [rows, 3*H*dh] (bf16), row t at position
    t mod S, with the first r dims of each head rotated by the fp32 cos / sin table [n_pos >= S, 2, r/2]
    (include/dalle_b200.h)."""
    rows, n_pos = _rope_args(qkv, table, H, dh, r, "rope_fwd")
    if S > n_pos:
        raise L.DB200Error(f"rope_fwd: period S {S} exceeds the table's {n_pos} positions")
    check(L.load().db200_rope_fwd(stream_ptr(), ptr(qkv), ptr(table), rows, int(S), H, dh, int(r)), "db200_rope_fwd")


def rope_bwd(dqkv, table, S, H, dh, r):
    """The transpose of rope_fwd in place on the dq and dk columns of dqkv [rows, 3*H*dh] (bf16)."""
    rows, n_pos = _rope_args(dqkv, table, H, dh, r, "rope_bwd")
    if S > n_pos:
        raise L.DB200Error(f"rope_bwd: period S {S} exceeds the table's {n_pos} positions")
    check(L.load().db200_rope_bwd(stream_ptr(), ptr(dqkv), ptr(table), rows, int(S), H, dh, int(r)), "db200_rope_bwd")


def rope_decode(qkv, table, pos, H, dh, r):
    """rope_fwd of one decoding step: every row of qkv [rows, 3*H*dh] at position pos (0 <= pos < n_pos)."""
    rows, n_pos = _rope_args(qkv, table, H, dh, r, "rope_decode")
    check(L.load().db200_rope_decode(stream_ptr(), ptr(qkv), ptr(table), rows, n_pos, H, dh, int(r), int(pos)),
          "db200_rope_decode")


def rope_decode_dev(qkv, table, pos_dev, H, dh, r):
    """rope_decode with the position read on the device from pos_dev (graph replay)."""
    rows, n_pos = _rope_args(qkv, table, H, dh, r, "rope_decode_dev")
    _chk(pos_dev, I32, "pos_dev")
    check(L.load().db200_rope_decode_dev(stream_ptr(), ptr(qkv), ptr(table), rows, n_pos, H, dh, int(r), ptr(pos_dev)),
          "db200_rope_decode_dev")


def _shift_rows(y, what):
    """(rows, d) of a contiguous bf16 [rows, d] operand of the token-shift kernels."""
    L.require_device()
    _chk(y, BF16, what)
    if not y.is_contiguous() or y.dim() != 2:
        raise L.DB200Error(f"{what}: expected a contiguous [rows, d] tensor, got {tuple(y.shape)}")
    return y.shape


def _shift_cache(cache, rows, d, what):
    """The length S of a token-shift cache bf16 [rows, S, d/2]."""
    _chk(cache, BF16, what)
    if not cache.is_contiguous() or cache.dim() != 3 or cache.shape[0] != rows or cache.shape[2] * 2 != d:
        raise L.DB200Error(f"{what}: expected a contiguous [{rows}, S, {d // 2}] cache, got {tuple(cache.shape)}")
    return cache.shape[1]


def shift_tokens_fwd(y, out, S, text_len, grid_w):
    """Token shift out = shift(y) of bf16 [rows, d] LayerNorm outputs, row t at position t mod S: the first d/4
    columns from the token above (image) or before (text), the next d/4 from the token to the left (image) or before
    (text), zeros where there is none (include/dalle_b200.h)."""
    rows, d = _shift_rows(y, "y")
    if tuple(_shift_rows(out, "out")) != (rows, d):
        raise L.DB200Error(f"shift_tokens_fwd: out {tuple(out.shape)} does not match y {(rows, d)}")
    check(L.load().db200_shift_tokens_fwd(stream_ptr(), ptr(y), ptr(out), rows, int(S), d, int(text_len),
                                          int(grid_w)), "db200_shift_tokens_fwd")


def shift_tokens_bwd(dout, dy, S, text_len, grid_w):
    """The transpose of shift_tokens_fwd: dy = shift^T(dout), bf16 [rows, d]."""
    rows, d = _shift_rows(dout, "dout")
    if tuple(_shift_rows(dy, "dy")) != (rows, d):
        raise L.DB200Error(f"shift_tokens_bwd: dy {tuple(dy.shape)} does not match dout {(rows, d)}")
    check(L.load().db200_shift_tokens_bwd(stream_ptr(), ptr(dout), ptr(dy), rows, int(S), d, int(text_len),
                                          int(grid_w)), "db200_shift_tokens_bwd")


def shift_tokens_decode(y, cache, pos, text_len, grid_w):
    """One decoding step of the token shift at position pos, in place on y bf16 [rows, d]: y's first d/2 columns go
    into cache[:, pos] (bf16 [rows, S, d/2]) and are replaced by the shifted chunks read from the cache."""
    rows, d = _shift_rows(y, "y")
    S = _shift_cache(cache, rows, d, "cache")
    check(L.load().db200_shift_tokens_decode(stream_ptr(), ptr(y), ptr(cache), rows, S, d, int(text_len), int(grid_w),
                                             int(pos)), "db200_shift_tokens_decode")


def shift_tokens_decode_dev(y, cache, pos_dev, text_len, grid_w):
    """shift_tokens_decode with the position read on the device from pos_dev (graph replay)."""
    rows, d = _shift_rows(y, "y")
    S = _shift_cache(cache, rows, d, "cache")
    _chk(pos_dev, I32, "pos_dev")
    check(L.load().db200_shift_tokens_decode_dev(stream_ptr(), ptr(y), ptr(cache), rows, S, d, int(text_len),
                                                 int(grid_w), ptr(pos_dev)), "db200_shift_tokens_decode_dev")


def shift_cache_fill(y, cache, P, rep=1):
    """Prefill hand-off of the token shift: y bf16 [B*P, d], the unshifted LayerNorm outputs of B prompts of P
    positions -> cache bf16 [B*rep, S, d/2], cache[b*rep + r, p] = y[b*P + p, :d/2] (kv_cache_fill's replica order)."""
    rows, d = _shift_rows(y, "y")
    if P < 1 or rows % P:
        raise L.DB200Error(f"shift_cache_fill: {rows} rows are not a whole number of {P}-position prompts")
    B = rows // P
    S = _shift_cache(cache, B * int(rep), d, "cache")
    check(L.load().db200_shift_cache_fill(stream_ptr(), ptr(y), ptr(cache), B, int(P), d, S, int(rep)),
          "db200_shift_cache_fill")


def _rope_emb_args(qkv, table, H, dh, what):
    """(rows, table positions, pairs) of a rotary_emb call after the dtype / shape checks."""
    L.require_device()
    _chk(qkv, BF16, what); _chk(table, F32, "table")
    if not qkv.is_contiguous() or qkv.dim() != 2 or qkv.shape[1] != 3 * H * dh:
        raise L.DB200Error(f"{what}: expected a contiguous [rows, {3 * H * dh}] q|k|v buffer, got {tuple(qkv.shape)}")
    if not table.is_contiguous() or table.dim() != 3 or table.shape[1] != 2 or not 1 <= table.shape[2] <= dh // 2:
        raise L.DB200Error(f"{what}: expected a contiguous [n_pos, 2, pairs <= {dh // 2}] table, got "
                           f"{tuple(table.shape)}")
    return qkv.shape[0], table.shape[0], table.shape[2]


def rope_emb_fwd(qkv, table, S, H, dh):
    """DALLE-pytorch's rotary embedding in place on every q, k and v head of qkv [rows, 3*H*dh] (bf16), row t at
    position t mod S: the interleaved pairs (2m, 2m+1), m < pairs, rotated by the fp32 cos / sin table
    [n_pos >= S, 2, pairs] (dalle_engine.rotary_emb_table; include/dalle_b200.h)."""
    rows, n_pos, pairs = _rope_emb_args(qkv, table, H, dh, "rope_emb_fwd")
    if S > n_pos:
        raise L.DB200Error(f"rope_emb_fwd: period S {S} exceeds the table's {n_pos} positions")
    check(L.load().db200_rope_emb_fwd(stream_ptr(), ptr(qkv), ptr(table), rows, int(S), H, dh, pairs),
          "db200_rope_emb_fwd")


def rope_emb_bwd(dqkv, table, S, H, dh):
    """The transpose of rope_emb_fwd in place on the dq, dk and dv columns of dqkv [rows, 3*H*dh] (bf16)."""
    rows, n_pos, pairs = _rope_emb_args(dqkv, table, H, dh, "rope_emb_bwd")
    if S > n_pos:
        raise L.DB200Error(f"rope_emb_bwd: period S {S} exceeds the table's {n_pos} positions")
    check(L.load().db200_rope_emb_bwd(stream_ptr(), ptr(dqkv), ptr(table), rows, int(S), H, dh, pairs),
          "db200_rope_emb_bwd")


def rope_emb_decode(qkv, table, pos, H, dh):
    """rope_emb_fwd of one decoding step: every row of qkv [rows, 3*H*dh] at position pos (0 <= pos < n_pos)."""
    rows, n_pos, pairs = _rope_emb_args(qkv, table, H, dh, "rope_emb_decode")
    check(L.load().db200_rope_emb_decode(stream_ptr(), ptr(qkv), ptr(table), rows, n_pos, H, dh, pairs, int(pos)),
          "db200_rope_emb_decode")


def rope_emb_decode_dev(qkv, table, pos_dev, H, dh):
    """rope_emb_decode with the position read on the device from pos_dev (graph replay)."""
    rows, n_pos, pairs = _rope_emb_args(qkv, table, H, dh, "rope_emb_decode_dev")
    _chk(pos_dev, I32, "pos_dev")
    check(L.load().db200_rope_emb_decode_dev(stream_ptr(), ptr(qkv), ptr(table), rows, n_pos, H, dh, pairs,
                                             ptr(pos_dev)), "db200_rope_emb_decode_dev")


def rows_repeat(src, dst, rep=1):
    """dst[b*rep + r] = src[b] for a [B, d] view src (rows may be strided, e.g. x.view(B, P, d)[:, P - 1])."""
    L.require_device()
    _chk(src, BF16, "src"); _chk(dst, BF16, "dst")
    B, d = src.shape
    assert dst.is_contiguous() and dst.shape[-1] == d and dst.numel() == B * int(rep) * d
    check(L.load().db200_rows_repeat(stream_ptr(), ptr(src), src.stride(0), ptr(dst), B, d, int(rep)),
          "db200_rows_repeat")
    return dst


def incr_i32(p, delta=1):
    L.require_device()
    check(L.load().db200_incr_i32(stream_ptr(), ptr(p), int(delta)), "db200_incr_i32")


def onehot_rows(idx, y, offset=0):
    L.require_device()
    _chk(idx, I32, "idx"); _chk(y, F32, "y")
    rows, K = y.shape
    check(L.load().db200_onehot_rows_f32(stream_ptr(), ptr(idx), ptr(y), rows, K, int(offset)), "db200_onehot_rows_f32")
    return y


# ----------------------------------------------------------------------------------------------- gMLP token mixing
def _sgu_act(t, what, C=None):
    """(rows, C) of a bf16 [rows, C] operand of the SGU kernels (rows may be strided, channels contiguous)."""
    L.require_device()
    _chk(t, BF16, what)
    if t.dim() != 2 or (C is not None and t.shape[1] != C):
        raise L.DB200Error(f"{what}: expected a [rows, {C if C is not None else 'C'}] tensor, got {tuple(t.shape)}")
    return t.shape


def _sgu_weight(w, n, what):
    _chk(w, BF16, what)
    if w.dim() != 2 or w.shape[0] < n or w.shape[1] < n:
        raise L.DB200Error(f"{what}: expected a [>= {n}, >= {n}] mixing weight, got {tuple(w.shape)}")


def sgu_mix_fwd(w, gn, res, c, h, mixed, B, n):
    """The SGU's token mixing over B sequences of n positions (include/dalle_b200.h): m = W[:n, :n] gn_b + c[i] in
    fp32, h = bf16(m * res), mixed = bf16(m) (or None).  gn, h, mixed contiguous bf16 [B n, C]; res [B n, C] with any
    row pitch (the first half of the proj_in output); w the bf16 weight, read through its pitch; c fp32 [>= n]."""
    rows, C = _sgu_act(gn, "gn")
    _sgu_act(res, "res", C); _sgu_act(h, "h", C); _chk(c, F32, "c")
    if mixed is not None:
        _sgu_act(mixed, "mixed", C)
    _sgu_weight(w, n, "w")
    if rows != B * n or not gn.is_contiguous() or not h.is_contiguous() or res.shape[0] != rows or \
            h.shape[0] != rows or (mixed is not None and (not mixed.is_contiguous() or mixed.shape[0] != rows)) or \
            c.numel() < n:
        raise L.DB200Error(f"sgu_mix_fwd: gn, h, mixed must be contiguous [{B * n}, {C}], res [{B * n}, {C}], c >= {n}")
    check(L.load().db200_sgu_mix_fwd(stream_ptr(), ptr(w), w.stride(0), ptr(gn), ptr(res), res.stride(0), ptr(c),
                                     ptr(h), ptr(mixed), B, n, C), "db200_sgu_mix_fwd")
    return h


def sgu_mix_dgrad(w, dmixed, dgn, B, n):
    """dgn_b = W[:n, :n]^T dmixed_b (bf16 [B n, C] contiguous)."""
    rows, C = _sgu_act(dmixed, "dmixed")
    _sgu_act(dgn, "dgn", C)
    _sgu_weight(w, n, "w")
    if rows != B * n or dgn.shape[0] != rows or not dmixed.is_contiguous() or not dgn.is_contiguous():
        raise L.DB200Error(f"sgu_mix_dgrad: dmixed and dgn must be contiguous [{B * n}, {C}]")
    check(L.load().db200_sgu_mix_dgrad(stream_ptr(), ptr(w), w.stride(0), ptr(dmixed), ptr(dgn), B, n, C),
          "db200_sgu_mix_dgrad")
    return dgn


def sgu_mix_wgrad(dmixed, gn, dw, B, n):
    """dw[i, j] (fp32 [n, n] view, any row pitch) += sum_b sum_c dmixed_b[i, c] gn_b[j, c] for j <= i; the strict upper
    triangle is never written."""
    rows, C = _sgu_act(dmixed, "dmixed")
    _sgu_act(gn, "gn", C)
    _chk(dw, F32, "dw")
    if rows != B * n or gn.shape[0] != rows or not dmixed.is_contiguous() or not gn.is_contiguous() or \
            dw.dim() != 2 or dw.shape[0] < n or dw.shape[1] < n:
        raise L.DB200Error(f"sgu_mix_wgrad: dmixed and gn must be contiguous [{B * n}, {C}], dw [>= {n}, >= {n}]")
    check(L.load().db200_sgu_mix_wgrad(stream_ptr(), ptr(dmixed), ptr(gn), ptr(dw), dw.stride(0), B, n, C),
          "db200_sgu_mix_wgrad")
    return dw


def sgu_bwd(dh, mixed, res, z_res, dmixed, du_res, dc, B, n):
    """The SGU's elementwise backward: dmixed = bf16(dh res), du_res = bf16(dh mixed gelu'(z_res)) (the res half of the
    proj_in gradient, any row pitch), dc[i] += sum over sequences and channels of dmixed at position i."""
    rows, C = _sgu_act(dh, "dh")
    for t, nm in ((mixed, "mixed"), (res, "res"), (z_res, "z_res"), (dmixed, "dmixed"), (du_res, "du_res")):
        _sgu_act(t, nm, C)
        if t.shape[0] != rows:
            raise L.DB200Error(f"sgu_bwd: {nm} has {t.shape[0]} rows, expected {rows}")
    _chk(dc, F32, "dc")
    if rows != B * n or dc.numel() < n or not (dh.is_contiguous() and mixed.is_contiguous() and dmixed.is_contiguous()):
        raise L.DB200Error(f"sgu_bwd: dh, mixed, dmixed must be contiguous [{B * n}, {C}], dc >= {n} entries")
    check(L.load().db200_sgu_bwd(stream_ptr(), ptr(dh), ptr(mixed), ptr(res), res.stride(0), ptr(z_res),
                                 z_res.stride(0), ptr(dmixed), ptr(du_res), du_res.stride(0), ptr(dc), B, n, C),
          "db200_sgu_bwd")


def sgu_gate_bwd(dgate, z_gate, du_gate):
    """du_gate = bf16(dgate gelu'(z_gate)): the gate half of the proj_in gradient (z_gate and du_gate any row pitch)."""
    rows, C = _sgu_act(dgate, "dgate")
    _sgu_act(z_gate, "z_gate", C); _sgu_act(du_gate, "du_gate", C)
    if not dgate.is_contiguous() or z_gate.shape[0] != rows or du_gate.shape[0] != rows:
        raise L.DB200Error(f"sgu_gate_bwd: dgate must be contiguous [{rows}, {C}], z_gate and du_gate [{rows}, {C}]")
    check(L.load().db200_sgu_gate_bwd(stream_ptr(), ptr(dgate), ptr(z_gate), z_gate.stride(0), ptr(du_gate),
                                      du_gate.stride(0), rows, C), "db200_sgu_gate_bwd")


def _sgu_decode_args(gn, res, w, c, cache, h):
    rows, C = _sgu_act(gn, "gn")
    _sgu_act(res, "res", C); _sgu_act(h, "h", C); _chk(c, F32, "c"); _chk(cache, BF16, "cache"); _chk(w, BF16, "w")
    if not cache.is_contiguous() or cache.dim() != 3 or cache.shape[0] != rows or cache.shape[2] != C:
        raise L.DB200Error(f"sgu_decode: expected a contiguous [{rows}, S, {C}] cache, got {tuple(cache.shape)}")
    S = cache.shape[1]
    if not gn.is_contiguous() or not h.is_contiguous() or res.shape[0] != rows or h.shape[0] != rows or \
            c.numel() < S or w.dim() != 2 or w.shape[0] < S or w.shape[1] < S:
        raise L.DB200Error(f"sgu_decode: gn and h contiguous [{rows}, {C}], res [{rows}, {C}], w [>= {S}, >= {S}], "
                           f"c >= {S} entries")
    return rows, S, C


def sgu_decode(gn, res, w, c, cache, h, pos):
    """One decoding step of the SGU at position pos: cache[:, pos] = gn, then h = bf16((sum_{j <= pos} w[pos, j]
    cache[:, j] + c[pos]) res) with the sum in fp32 in j order."""
    rows, S, C = _sgu_decode_args(gn, res, w, c, cache, h)
    check(L.load().db200_sgu_decode(stream_ptr(), ptr(gn), ptr(res), res.stride(0), ptr(w), w.stride(0), ptr(c),
                                    ptr(cache), ptr(h), rows, S, C, int(pos)), "db200_sgu_decode")
    return h


def sgu_decode_dev(gn, res, w, c, cache, h, pos_dev):
    """sgu_decode with the position read on the device from pos_dev (graph replay)."""
    rows, S, C = _sgu_decode_args(gn, res, w, c, cache, h)
    _chk(pos_dev, I32, "pos_dev")
    check(L.load().db200_sgu_decode_dev(stream_ptr(), ptr(gn), ptr(res), res.stride(0), ptr(w), w.stride(0), ptr(c),
                                        ptr(cache), ptr(h), rows, S, C, ptr(pos_dev)), "db200_sgu_decode_dev")
    return h


def sgu_cache_fill(gn, cache, P, rep=1):
    """Prefill hand-off of the SGU: gn bf16 [B*P, C] -> cache bf16 [B*rep, S, C], cache[b*rep + r, p] = gn[b*P + p]
    (kv_cache_fill's replica order)."""
    rows, C = _sgu_act(gn, "gn")
    _chk(cache, BF16, "cache")
    if P < 1 or rows % P or not gn.is_contiguous():
        raise L.DB200Error(f"sgu_cache_fill: {rows} contiguous rows are not a whole number of {P}-position prompts")
    B = rows // P
    if not cache.is_contiguous() or cache.dim() != 3 or cache.shape[0] != B * int(rep) or cache.shape[2] != C:
        raise L.DB200Error(f"sgu_cache_fill: expected a contiguous [{B * int(rep)}, S, {C}] cache, got "
                           f"{tuple(cache.shape)}")
    check(L.load().db200_sgu_cache_fill(stream_ptr(), ptr(gn), ptr(cache), B, int(P), C, cache.shape[1], int(rep)),
          "db200_sgu_cache_fill")
