/* dalle_b200.h — C ABI of libdalle_b200.so (hand-written sm_90a kernels for the DALL-E / dVAE training hot path).
 *
 * The reference (EleutherAI/DALLE-mtf) has no FFI: its arithmetic is executed by mesh-tensorflow / TensorFlow ops
 * called from Python graph-building code.  Each entry point below replaces the library call(s) the reference makes
 * at the cited file:line (paths relative to the reference root), so a maintainer can bind it with ctypes in place of
 * that call (see INTEGRATION.md).
 *
 * Conventions
 *   - every function returns int: 0 = DB200_OK, negative = error; db200_last_error() gives a thread-local message.
 *     Nothing throws, nothing calls exit().  Shape / alignment violations are checked and reported.
 *   - all tensor pointers are raw DEVICE pointers owned by the caller (PyTorch); row-major, innermost dim contiguous,
 *     16-byte aligned.  The library never allocates or frees device memory and keeps no pointers across calls.
 *   - reductions over many CTAs are never float atomics: each CTA stores a partial into a scratch WORKSPACE the caller
 *     passes in (its size comes from the matching db200_*_workspace_bytes query, which depends on the shape and the
 *     device's SM count), and the partials are added in a fixed order on the same stream, so results are identical
 *     from run to run.  A workspace may be reused as soon as the call's work on that stream has finished.
 *   - `stream` is a cudaStream_t (CUstream) passed as void*; kernels are enqueued on it and the call returns
 *     without synchronising.
 *   - bf16 = __nv_bfloat16 (2 bytes).  "f32" = IEEE float.
 */
#ifndef DALLE_B200_H_
#define DALLE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DB200_OK 0
#define DB200_E_INVALID (-1)     /* bad shape / argument */
#define DB200_E_ALIGN (-2)       /* pointer or leading dimension not 16-byte aligned */
#define DB200_E_CUDA (-3)        /* CUDA runtime / driver error (message has the string) */
#define DB200_E_UNSUPPORTED (-4) /* valid request the kernels do not cover (e.g. head_dim not in {64,128}) */

typedef void* db200_stream_t;

const char* db200_last_error(void);
int db200_version(void);
/* number of kernels this library has launched in this process (monotonic; used for bench.py's gpu_launches) */
unsigned long long db200_launch_count(void);
/* 0 if the current CUDA device is compute capability 9.0 (sm_90a cubins can run), else DB200_E_UNSUPPORTED. */
int db200_device_check(void);

/* ------------------------------------------------------------------------------------------------------------------
 * K1  token + position embedding.   Replaces mtf.gather(wte, ids) + mtf.gather(wpe, range) + add
 *     src/dalle_mtf/models.py:186-219.   out[b,s,:] = wte[ids[b,s],:] + wpe[s,:]
 *     bwd: dwte[ids[b,s],:] += dx[b,s,:]   (order-independent: 64-bit fixed point),  dwpe[s,:] += sum_b dx[b,s,:]
 * ------------------------------------------------------------------------------------------------------------------ */
int db200_embed_fwd(db200_stream_t stream, const int32_t* ids, const void* wte_bf16, const void* wpe_bf16,
                    void* out_bf16, int B, int S, int d, int V);
/* embed_bwd sums dwte rows in 64-bit fixed point (2^-40 resolution, |sum| < 8.4e6) in the workspace: integer addition
 * does not depend on the order in which tokens with the same id arrive. */
int db200_embed_bwd(db200_stream_t stream, const int32_t* ids, const void* dx_bf16, float* dwte, float* dwpe, int B,
                    int S, int d, int V, void* workspace, int64_t workspace_bytes);
int64_t db200_embed_bwd_workspace_bytes(int d, int V);

/* T0 token assembly: tokens[b] = concat(text_ids[b], image_idx[b] + image_offset).  Replaces tf.concat at
 * src/model_fns.py:117-122 (image_offset = text_vocab_size). */
int db200_assemble_tokens(db200_stream_t stream, const int32_t* text_ids, const int32_t* image_idx, int32_t* tokens,
                          int B, int text_len, int image_len, int image_offset);

/* label shift: labels[b][t] = ids[b][t+1], labels[b][S-1] = eos_id.  Replaces the pad + gather at
 * src/dalle_mtf/models.py:407-410 (pad op: src/dalle_mtf/ops.py:6-68). */
int db200_shift_labels(db200_stream_t stream, const int32_t* ids, int32_t* labels, int B, int S, int eos_id);

/* ------------------------------------------------------------------------------------------------------------------
 * K2  LayerNorm.   Replaces DALLE.layer_norm + norm():  src/dalle_mtf/models.py:373-389, src/dalle_mtf/layers.py:30-33
 *     y = (x - mean) * rsqrt(mean((x-mean)^2) + eps) * g + b      (biased variance, fp32 statistics)
 *     bwd: dx = [dres +] LN'(dy);  dg += sum_rows dy*xhat;  db += sum_rows dy   (dg/db accumulate, fp32)
 * ------------------------------------------------------------------------------------------------------------------ */
int db200_layernorm_fwd(db200_stream_t stream, const void* x_bf16, const float* g, const float* b, void* y_bf16,
                        float* mean, float* rstd, int rows, int d, float eps);
int db200_layernorm_bwd(db200_stream_t stream, const void* dy_bf16, const void* x_bf16, const float* g,
                        const float* mean, const float* rstd, const void* dres_bf16_or_null, void* dx_bf16, float* dg,
                        float* db, int rows, int d, void* workspace, int64_t workspace_bytes);
/* same, and additionally dxsum[c] += sum_rows dx[row][c]: the bias gradient of the linear layer whose output
 * gradient dx is (fuses the column-sum pass; dxsum may be NULL) */
int db200_layernorm_bwd_ex(db200_stream_t stream, const void* dy_bf16, const void* x_bf16, const float* g,
                           const float* mean, const float* rstd, const void* dres_bf16_or_null, void* dx_bf16,
                           float* dg, float* db, float* dxsum_or_null, int rows, int d, void* workspace,
                           int64_t workspace_bytes);
int64_t db200_layernorm_bwd_workspace_bytes(int rows, int d);

/* ------------------------------------------------------------------------------------------------------------------
 * K3/K5/K6/K8  bf16 GEMM on wgmma (TMA-fed, register accumulators, fp32 accumulate):   D[M,N] = A[M,K] * B[K,N]
 *     Replaces every mtf einsum / mtf.layers.dense on the path: q/k/v/o projections src/dalle_mtf/models.py:235-244,
 *     303-311; MLP :317-324, 361-371; to_logits :391-395; and their mtf.gradients (src/optimizers.py:34).
 *   Operand storage:  a_mn_major = 0: A stored [M][K] (lda = row pitch in elements);  1: A stored [K][M].
 *                     b_mn_major = 0: B stored [N][K];                                  1: B stored [K][N].
 *   (forward x*W: A k-major, B mn-major;  dgrad dy*W^T: both k-major;  wgrad x^T*dy: both mn-major.)
 * ------------------------------------------------------------------------------------------------------------------ */
enum {
  DB200_EPI_STORE = 0,    /* D = act(alpha*acc + bias[n]) + residual[m,n]  -> bf16 or f32                          */
  DB200_EPI_ATOMIC = 1,   /* D(f32) += alpha*acc  (gradient accumulation; split-K slices summed in split order)   */
  DB200_EPI_RELU_BWD = 2, /* D(bf16) = alpha*acc * (aux[m,n] > 0)          (backward of the MLP's ReLU)            */
  DB200_EPI_CE_STATS = 3, /* no D: per (row, n-tile) max & sum-exp of acc+bias over valid columns + label logit    */
  DB200_EPI_CE_GRAD = 4   /* D(bf16) = alpha * (exp(acc+bias - lse[m]) - [n == label[m]]), 0 for n >= n_valid; alpha > 0 */
};

typedef struct db200_gemm_epilogue {
  int32_t mode;         /* DB200_EPI_*                                                            */
  int32_t out_f32;      /* STORE only: 1 -> D is float, 0 -> D is bf16                            */
  int32_t relu;         /* STORE only                                                             */
  int32_t split_k;      /* ATOMIC only: number of K splits (>=1); other modes must pass 1         */
  float alpha;          /* scale applied to the accumulator                                       */
  const float* bias;    /* [N] f32 or NULL                                                        */
  const void* residual; /* bf16 [M][ldr] or NULL (STORE)                                          */
  int64_t ldr;
  const void* aux;      /* bf16 [M][ldaux] (RELU_BWD)                                             */
  int64_t ldaux;
  const int32_t* labels; /* [M]  (CE_*)                                                           */
  float* part_max;       /* [n_tiles][M] (CE_STATS)   n_tiles = db200_gemm_ce_tiles(N)              */
  float* part_sum;       /* [n_tiles][M] (CE_STATS)                                               */
  float* label_logit;    /* [M] (CE_STATS)                                                        */
  const float* lse;      /* [M] (CE_GRAD)                                                         */
  int32_t n_valid;       /* CE_*: number of real vocabulary columns (<= N)                        */
  int32_t reserved;
  float* colsum;         /* CE_GRAD / RELU_BWD: colsum[n] += sum_m D[m][n] (fused bias gradient) or NULL */
  void* workspace;       /* device scratch of db200_gemm_workspace_bytes() bytes (16-byte aligned), or NULL when 0 */
  int64_t workspace_bytes;
} db200_gemm_epilogue;

int db200_gemm_bf16(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda, const void* B, int b_mn_major,
                    int64_t ldb, void* D, int64_t ldd, int M, int N, int K, const db200_gemm_epilogue* epi);
/* number of N tiles the CE_STATS epilogue writes per row for a given N (host helper for sizing part_max/part_sum) */
int db200_gemm_ce_tiles(int N);
/* epi->workspace size for this product: split-K slices (ATOMIC) or fused column sums (CE_GRAD / RELU_BWD with colsum) */
int64_t db200_gemm_workspace_bytes(int M, int N, int K, const db200_gemm_epilogue* epi);

/* ------------------------------------------------------------------------------------------------------------------
 * K7  cross-entropy pieces around the vocabulary GEMM (logits never reach HBM in fp32).
 *     Replaces mtf.layers.softmax_cross_entropy_with_logits + reduce_mean: src/dalle_mtf/models.py:348-359.
 *     ce_finish:  lse[m] = logsumexp over tiles;  loss_rows[m] = lse[m] - label_logit[m];  *loss_sum += sum_m loss_rows
 * ------------------------------------------------------------------------------------------------------------------ */
int db200_ce_finish(db200_stream_t stream, const float* part_max, const float* part_sum, const float* label_logit,
                    float* lse, float* loss_rows, float* loss_sum, int M, int n_tiles, void* workspace,
                    int64_t workspace_bytes);
int64_t db200_ce_finish_workspace_bytes(int M);

/* ------------------------------------------------------------------------------------------------------------------
 * K4  causal flash attention on wgmma.  Replaces mtf_transformer.attention.attention with the [S,S] -1e10 mask:
 *     src/dalle_mtf/models.py:221-227, 287-299.   qkv: bf16 [B][S][3][H][dh] (output of the fused q|k|v GEMM),
 *     out: bf16 [B][S][H][dh],  lse: f32 [B][H][S] (natural-log sum-exp of scale*q.k).  Reference scale = 1.0.
 *     bwd: dqkv same layout as qkv; dq_accum f32 [B][S][H][dh] and delta f32 [B][H][S] are caller workspaces.
 * ------------------------------------------------------------------------------------------------------------------ */
int db200_attn_causal_fwd(db200_stream_t stream, const void* qkv_bf16, void* out_bf16, float* lse, int B, int S,
                          int H, int dh, float scale);
int db200_attn_causal_bwd(db200_stream_t stream, const void* qkv_bf16, const void* out_bf16, const void* dout_bf16,
                          const float* lse, float* dq_accum, float* delta, void* dqkv_bf16, int B, int S, int H,
                          int dh, float scale);

/* ------------------------------------------------------------------------------------------------------------------
 * small HBM-bound helpers
 * ------------------------------------------------------------------------------------------------------------------ */
/* out[c] += sum_r x[r][c]   (bias gradients) */
int db200_colsum_bf16(db200_stream_t stream, const void* x_bf16, int64_t ld, int rows, int cols, float* out_accum,
                      void* workspace, int64_t workspace_bytes);
int64_t db200_colsum_workspace_bytes(int rows, int cols);
int db200_cast_f32_to_bf16(db200_stream_t stream, const float* src, void* dst_bf16, size_t n);
int db200_cast_bf16_to_f32(db200_stream_t stream, const void* src_bf16, float* dst, size_t n);
/* hi = bf16(x), lo = bf16(x - hi) (lo may be NULL): an fp32 operand as two bf16 tensor-core operands */
int db200_split_f32_to_bf16x2(db200_stream_t stream, const float* src, void* hi_bf16, void* lo_bf16_or_null, size_t n);

/* ------------------------------------------------------------------------------------------------------------------
 * K9/K10  optimiser.  Replaces clip_by_global_norm src/optimizers.py:11-16 and
 *     mtf.optimize.AdamWeightDecayOptimizer.apply_grad (math restated in-tree at src/optimizers.py:128-172), and,
 *     with bias_correction=1, tf.train.AdamOptimizer as used by src/model_fns_tf.py:58-66.
 *   sqnorm:  *out_accum += sum g^2        (caller zeroes out_accum)
 *   adam:    gs = g * grad_scale * (clip>0 ? clip / max(sqrt(*gnorm_sq)*grad_scale, clip) : 1)
 *            m = b1*m + (1-b1)*gs;  v = b2*v + (1-b2)*gs^2
 *            bias_correction == 0:  p -= lr * (m / (sqrt(v) + eps) + wd*p)
 *            bias_correction == 1:  p -= lr*sqrt(1-b2^t)/(1-b1^t) * m / (sqrt(v) + eps)      (t = step, >= 1)
 *            p_bf16 (optional) receives the rounded updated parameter (compute copy).
 *            zero_grad != 0: g is overwritten with 0 once consumed (the gradient buffer accumulates (+=), so it
 *            must start every step at zero: this folds that memset into the pass that already streams g).
 * ------------------------------------------------------------------------------------------------------------------ */
int db200_sqnorm_f32(db200_stream_t stream, const float* g, size_t n, float* out_accum, void* workspace,
                     int64_t workspace_bytes);
int64_t db200_sqnorm_workspace_bytes(size_t n);
int db200_adam_step(db200_stream_t stream, float* p, float* m, float* v, float* g, void* p_bf16_or_null,
                    size_t n, float lr, float beta1, float beta2, float eps, float weight_decay,
                    const float* gnorm_sq_or_null, float clip, float grad_scale, int bias_correction, int step,
                    int zero_grad);

/* ------------------------------------------------------------------------------------------------------------------
 * K11  discrete-VAE convolutions, NHWC activations / HWIO kernels like tf.layers.conv2d
 *     (src/vae_tf/models.py:95-109, 139-155).  Shared-memory-staged direct convolutions (no im2col buffer).
 *     conv2d:            y = conv(x, w[kh][kw][cin][cout], stride, SAME) + bias  [relu: ReLU on the output]
 *                        [+ residual]                                     x: [N][H][W][Cin]  y: [N][Ho][Wo][Cout]
 *     conv2d_transpose:  tf.layers.conv2d_transpose(k=4, s=2, SAME), kernel [kh][kw][cout][cin]
 *     *_dgrad / *_wgrad: gradients w.r.t. input / kernel+bias (dw, dbias accumulate in f32).
 *   Activations are bf16 or f32 (act_f32 flag), parameters f32, accumulation f32.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct db200_conv_desc {
  int32_t N, H, W, Cin;   /* input  */
  int32_t Ho, Wo, Cout;   /* output */
  int32_t KH, KW, stride; /* SAME padding: pad_top = max((Ho-1)*stride + KH - H, 0) / 2 */
  int32_t transposed;     /* 1 -> conv2d_transpose geometry (x is the low-res tensor [N][H][W][Cin]) */
  int32_t act_f32;        /* 1 -> activations are float, 0 -> bf16 */
  int32_t relu;           /* fwd: apply ReLU to the output (fuses the residual block's activation, models.py:102) */
  int32_t reserved;
} db200_conv_desc;

int db200_conv2d_fwd(db200_stream_t stream, const db200_conv_desc* c, const void* x, const float* w,
                     const float* bias_or_null, const void* residual_or_null, void* y);
/* Tensor-core paths (wgmma implicit GEMM; 4-D TMA boxes per filter tap, no im2col), bf16 NHWC activations, bf16
 * kernels (same memory layout as the f32 kernels: HWIO, or [kh][kw][out][in] for conv2d_transpose), f32 bias / dw.
 *   fwd_tc   : conv or conv2d_transpose forward; needs Cin % 64 == 0, Cout % 8 == 0
 *   dgrad_tc : needs Cout % 64 == 0, Cin % 8 == 0; optional ReLU mask (dx *= x_mask > 0) and residual-gradient add
 *   wgrad_tc : dw (f32) += ...; needs Cin % 64 == 0 and Cout % 64 == 0; bias gradient = db200_colsum_bf16 of dy
 * Stride 1 or 2 (even H, W).  Unsupported shapes return DB200_E_UNSUPPORTED: callers pick the direct kernels
 * explicitly, there is no silent fallback. */
int db200_conv2d_fwd_tc(db200_stream_t stream, const db200_conv_desc* c, const void* x_bf16, const void* w_bf16,
                        const float* bias_or_null, const void* residual_bf16_or_null, void* y_bf16);
int db200_conv2d_dgrad_tc(db200_stream_t stream, const db200_conv_desc* c, const void* dy_bf16, const void* w_bf16,
                          const void* x_mask_bf16_or_null, const void* dres_bf16_or_null, void* dx_bf16);
int db200_conv2d_wgrad_tc(db200_stream_t stream, const db200_conv_desc* c, const void* x_bf16, const void* dy_bf16,
                          float* dw);
/* First encoder layer (Cin = 3, 4x4, stride 2, SAME) straight from the fp32 image to bf16 activations:
 * dedicated CUDA-core kernel (K = 48 is too small for the tensor pipe).  x: f32 [N][H][W][3], w: f32 [4][4][3][Cout]. */
int db200_conv2d_first_fwd(db200_stream_t stream, const float* x, const float* w, const float* bias_or_null,
                           void* y_bf16, int N, int H, int W, int Cout);
/* the same layer on the CUDA cores (fp32 FMA): kept for A/B measurements only */
int db200_conv2d_first_fwd_fma(db200_stream_t stream, const float* x, const float* w, const float* bias_or_null,
                           void* y_bf16, int N, int H, int W, int Cout);
int db200_conv2d_dgrad(db200_stream_t stream, const db200_conv_desc* c, const void* dy, const float* w,
                       const void* x_for_relu_mask_or_null, const void* dres_or_null, void* dx);
int db200_conv2d_wgrad(db200_stream_t stream, const db200_conv_desc* c, const void* x, const void* dy, float* dw,
                       float* dbias_or_null);

/* ------------------------------------------------------------------------------------------------------------------
 * K12/K13  codebook matmul + Gumbel-softmax + argmax  (src/vae_tf/models.py:111-120,124-127; src/vae_tf/layers.py:4-21;
 *          src/model_fns.py:76).  All f32, rows = N*h*w positions, K codes.
 *   rowmatmul:        out[r][n] = sum_k a[r][k] * b[k][n]   (or b^T) — small-K f32 matmul used for the codebook
 *   gumbel_softmax:   y = softmax((logits - log(-log u)) / tau);  hard: y_out = onehot(argmax y) (first max wins)
 *   gumbel_softmax_bwd: dlogits = (y .* (dy - sum(dy.*y))) / tau      (straight-through: dy is taken w.r.t. y_out)
 *   argmax_rows:      idx[r] = first index of the row maximum (tf.math.argmax tie rule)
 * ------------------------------------------------------------------------------------------------------------------ */
int db200_rowmatmul_f32(db200_stream_t stream, const float* a, const float* b, float* out, int rows, int K, int N,
                        int b_transposed, int accumulate);
int db200_rowmatmul_tn_f32(db200_stream_t stream, const float* a, const float* b, float* out_accum, int rows, int M,
                           int N); /* out[M][N] += a[rows][M]^T * b[rows][N] */
int db200_gumbel_softmax_fwd(db200_stream_t stream, const float* logits, const float* u_or_null, float* y_soft,
                             float* y_out, int32_t* idx_or_null, int rows, int K, float tau, int hard);
int db200_gumbel_softmax_bwd(db200_stream_t stream, const float* y_soft, const float* dy, float* dlogits, int rows,
                             int K, float tau);
int db200_argmax_rows_f32(db200_stream_t stream, const float* x, int32_t* idx, int rows, int K);
/* mse:  *loss_accum += sum((a-b)^2) * scale;  dgrad: da = 2*(a-b)*scale */
int db200_mse_fwd_bwd(db200_stream_t stream, const float* pred, const float* target, float* dpred_or_null,
                      float* loss_accum, size_t n, float scale);

/* ------------------------------------------------------------------------------------------------------------------
 * N2/N3  data formats either side of the step ("next" rows of SURVEY.md section 8f).
 *   Host-memory functions (no CUDA): CRC-32C, TFRecord framing / indexing.  Replace tf.io.TFRecordWriter
 *   (src/data/create_tfrecords.py:153-178) and tf.data.TFRecordDataset (src/input_fns.py:80,116).
 *     record = u64le length | u32le masked_crc(length bytes) | data | u32le masked_crc(data)
 *     masked_crc(x) = rotr15(crc32c(x)) + 0xa282ead8
 *   db200_tfrecord_index: payload offsets / lengths of every record in a file image; *n_records = records found (may
 *   exceed max_records: call again with larger arrays); truncated / corrupt input is DB200_E_INVALID.
 * ------------------------------------------------------------------------------------------------------------------ */
int db200_crc32c(const void* data, uint64_t n, uint32_t* crc_out);
int db200_tfrecord_masked_crc(const void* data, uint64_t n, uint32_t* crc_out);
int db200_tfrecord_frame(const void* data, uint64_t n, void* out_n_plus_16_bytes);
int db200_tfrecord_index(const void* buf, uint64_t n, int verify_crc, uint64_t* offsets, uint64_t* lengths,
                         uint64_t max_records, uint64_t* n_records);
/* Batch of decoded uint8 HWC images (concatenated in `packed`, image b at byte offsets[b], heights[b] x widths[b] x
 * channels) -> out f32 NHWC [batch][out_size][out_size][channels] = (crop_and_resize(img, boxes[b]) - 127.5) / 127.5
 * with TensorFlow's bilinear CropAndResize semantics (extrapolation value 0).  boxes[b] = {y1, x1, y2, x2} normalised.
 * Replaces decode_img's tf.image.crop_and_resize + scaling, src/input_fns.py:4-21.  All pointers are device pointers. */
int db200_image_crop_resize_normalize(db200_stream_t stream, const uint8_t* packed, const int64_t* offsets,
                                      const int32_t* heights, const int32_t* widths, const float* boxes, float* out,
                                      int batch, int channels, int out_size);

/* ------------------------------------------------------------------------------------------------------------------
 * N4  incremental decoding with a K/V cache ("next" row of SURVEY.md section 8f): the path the reference sketches with
 *     is_incremental_inference / context (src/dalle_mtf/models.py:246-254, 281-285) but leaves unreachable
 *     (PREDICT raises NotImplementedError, src/model_fns.py:135-136).
 *   embed_fwd_at : out[b,:] = wte[ids[b],:] + wpe[pos,:]                                       (bf16, one position)
 *   attn_decode  : qkv_step bf16 [B][3][H][dh] = this position's q|k|v; k,v are written into k_cache / v_cache
 *                  (bf16 [B][S][H][dh]) at `pos`, then out[b,h,:] = softmax_{j<=pos}(scale q.k_j) v_j  (bf16 [B][H][dh])
 *   sample_rows  : idx[r] = lo + argmax_{lo<=c<hi}(logits[r][c] * inv_temp - log(-log(u[r][c-lo]))), first maximum;
 *                  u NULL = greedy.  logits f32 [rows][ld], u f32 [rows][hi-lo] uniform in (0,1).
 *   onehot_rows  : y[r][c] = (c == idx[r] - offset), f32 [rows][K]   (input of the tied codebook matmul,
 *                  src/vae_tf/models.py:127, when decoding sampled image tokens)
 * ------------------------------------------------------------------------------------------------------------------ */
int db200_embed_fwd_at(db200_stream_t stream, const int32_t* ids, const void* wte_bf16, const void* wpe_bf16,
                       void* out_bf16, int B, int d, int V, int n_positions, int pos);
int db200_attn_decode(db200_stream_t stream, const void* qkv_step_bf16, void* k_cache_bf16, void* v_cache_bf16,
                      void* out_bf16, int B, int S, int H, int dh, int pos, float scale);
int db200_sample_rows(db200_stream_t stream, const float* logits, const float* u_or_null, int32_t* idx, int rows,
                      long long ld, int lo, int hi, float inv_temp);
int db200_onehot_rows_f32(db200_stream_t stream, const int32_t* idx, float* y, int rows, int K, int offset);
/* Device-side-position variants: the position lives in ONE int32 in device memory (`pos_dev`, advanced with
 * db200_incr_i32), so a single captured CUDA graph of the per-position step is replayed for every position (generation
 * is launch-bound: ~46 kernels per position).  `tokens` is the [B][ld] token matrix: the step reads column *pos_dev and
 * the sampler writes column *pos_dev + 1. */
int db200_embed_fwd_at_dev(db200_stream_t stream, const int32_t* tokens, long long ld, const void* wte_bf16,
                           const void* wpe_bf16, void* out_bf16, int B, int d, int V, const int32_t* pos_dev);
int db200_attn_decode_dev(db200_stream_t stream, const void* qkv_step_bf16, void* k_cache_bf16, void* v_cache_bf16,
                          void* out_bf16, int B, int S, int H, int dh, const int32_t* pos_dev, float scale);
int db200_sample_rows_at(db200_stream_t stream, const float* logits, const float* u_or_null, int32_t* tokens,
                         long long ld_tokens, int rows, long long ld, int lo, int hi, float inv_temp,
                         const int32_t* pos_dev);
int db200_incr_i32(db200_stream_t stream, int32_t* p, int delta);

/* Segmented bf16 -> f32 gather (one launch): segment i copies table[3i+2] elements from src + table[3i] to
 * dst + table[3i+1]; `table_dev` is an int64 array in device memory.  ZeRO-1 mode: rebuilds the compact fp32 copy of the
 * vector parameters (LayerNorm g/b, biases) from the all-gathered bf16 parameters (mtf casts every variable to the
 * activation dtype when it is used, src/dalle_mtf/ops.py:76-82). */
int db200_gather_cast_bf16_f32(db200_stream_t stream, const void* src_bf16, float* dst, const int64_t* table_dev,
                               int n_segments);

/* tf.space_to_depth (inverse = 0) / tf.depth_to_space (inverse = 1), f32 NHWC, block size s: the `stack_factor`
 * re-packing of the VAE's input and output (src/vae_tf/models.py:85-86, 155-161).  H, W, C describe the FLAT image:
 * deep[n, y, x, (dy*s + dx)*C + c] = flat[n, y*s + dy, x*s + dx, c]. */
int db200_space_to_depth_f32(db200_stream_t stream, const float* in, float* out, int N, int H, int W, int C, int s,
                             int inverse);

/* ------------------------------------------------------------------------------------------------------------------
 * D1  data-parallel collectives: hand-driven NCCL over NVLink / NVSwitch behind the C ABI.
 *     Replaces the all-reduce mesh-tensorflow inserts for every weight gradient when it lowers the graph
 *     (src/optimizers.py:34 mtf.gradients + src/model_fns.py:189 mtf.Lowering; layout "batch_dim:data",
 *     configs/dalle_example.json:20-21) and tf.tpu.CrossShardOptimizer's gradient mean (src/model_fns_tf.py:61).
 *   One process per GPU.  db200_comm owns an ncclComm_t, a high-priority communication stream and two events.
 *   comm_load_nccl    : dlopen libnccl (path of the library to use, or NULL for "libnccl.so.2"); called implicitly.
 *   comm_unique_id    : ncclGetUniqueId into a caller buffer (>= 128 bytes); rank 0 creates it, the host code ships it
 *                       to the other ranks (any side channel), every rank then calls comm_create.
 *   comm_create       : ncclCommInitRankConfig on `device`; max_ctas > 0 caps the CTAs NCCL may occupy so that the
 *                       persistent wgmma GEMM grids running concurrently keep their SMs (0 = NCCL's default).
 *   comm_register     : ncclCommRegister of a long-lived buffer (the flat gradient buffer); best effort.
 *   bucket_allreduce_launch : in-place SUM all-reduce of buf[0..count) (dtype DB200_F32 / DB200_BF16) on the comm
 *                       stream, ordered after everything already enqueued on compute_stream; does not block it.
 *   bucket_reduce_scatter_launch / bucket_all_gather_launch : the ZeRO-1 pair (optimiser-state sharding): recv/send
 *                       hold count_per_rank elements per rank.
 *   bucket_allreduce_wait   : compute_stream waits (on the device; no host block) for every collective launched so far.
 * ------------------------------------------------------------------------------------------------------------------ */
#define DB200_F32 0
#define DB200_BF16 1
/* Persistent kernels size their grids to (SM count - n): leaves n SMs to a collective that runs concurrently (the
 * data-parallel path reserves the CTA cap it gave NCCL).  0 <= n <= 64; process-wide. */
int db200_set_reserved_sms(int n);
typedef struct db200_comm db200_comm;
int db200_comm_load_nccl(const char* libnccl_path);
int db200_comm_unique_id(void* id_out, size_t bytes);
int db200_comm_create(int device, int rank, int world, const void* unique_id, int max_ctas, db200_comm** out);
int db200_comm_destroy(db200_comm* comm);
int db200_comm_register(db200_comm* comm, void* buf, size_t bytes, int* registered);
int db200_comm_info(db200_comm* comm, int* rank, int* world, int* nccl_version);
int db200_bucket_allreduce_launch(db200_comm* comm, db200_stream_t compute_stream, void* buf, size_t count, int dtype);
int db200_bucket_reduce_scatter_launch(db200_comm* comm, db200_stream_t compute_stream, const void* send, void* recv,
                                       size_t count_per_rank, int dtype);
int db200_bucket_all_gather_launch(db200_comm* comm, db200_stream_t compute_stream, const void* send, void* recv,
                                   size_t count_per_rank, int dtype);
int db200_bucket_allreduce_wait(db200_comm* comm, db200_stream_t compute_stream);

#ifdef __cplusplus
}
#endif
#endif /* DALLE_B200_H_ */
