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
 * D0  dropout masks.  Replaces mtf.dropout at src/dalle_mtf/models.py:198-200, 215-217, 312-314, 321-323 and the
 *     dropout_rate of mtf_transformer.attention.attention at :290-299.  No mask is ever stored: the kernels that
 *     apply a mask regenerate it from a counter-based generator (Philox4x32-10), so a keep decision is a pure function
 *     of (seed, step, site, global element index):
 *       key = (lo32(seed), hi32(seed)),  counter = (lo32(n), hi32(n), site, step),  the element reads word w
 *       elementwise [rows][cols], row 0 = global row row0:  e = (row0 + r) * cols + c,  n = e >> 2,  w = e & 3
 *       attention weights (b, h, i, j), b = row0 + local sequence index, S2 = ceil(S / 2):
 *                                 n = ((b * H + h) * S2 + i / 2) * S2 + j / 2,  w = 2 * (i & 1) + (j & 1)
 *       keep iff word >= threshold (= floor(rate * 2^32)); kept values are multiplied by scale (= 1 / (1 - rate)).
 *       caption dropout (site DB200_SITE_CAPTION, db200_assemble_tokens_ex): one decision per sequence, the
 *                                 elementwise layout with cols = 1, e = row0 + b; the caption is dropped iff
 *                                 word < threshold.
 *     Every entry point that takes a `const db200_dropout*` treats NULL, or threshold 0, as "no dropout" and then runs
 *     exactly the kernels of the entry point without dropout.
 * ------------------------------------------------------------------------------------------------------------------ */
#define DB200_SITE_CAPTION 0xFFFFFFFFu /* above every layer site 2+3l .. 4+3l of a model with fewer than 2^30 layers */
typedef struct db200_dropout {
  uint64_t seed;
  uint32_t step;      /* global optimiser step */
  uint32_t site;      /* wte 0, wpe 1; layer l: attention weights 2+3l, attention output 3+3l, MLP output 4+3l;
                         caption DB200_SITE_CAPTION */
  uint32_t threshold; /* floor(rate * 2^32) */
  float scale;        /* 1 / (1 - rate) */
  int64_t row0;       /* elementwise: global row of row 0; attention: global sequence index of sequence 0 */
} db200_dropout;

#define DB200_DROPOUT_ELEMENTWISE 0 /* dims: rows, cols (cols % 4 == 0)     keep: uint8 [rows][cols]   */
#define DB200_DROPOUT_ATTENTION 1   /* dims: B, H, S                         keep: uint8 [B][H][S][S]   */
/* keep[...] = 1 where the element is kept, 0 where it is dropped (tests and oracle comparisons). */
int db200_dropout_mask(db200_stream_t stream, const db200_dropout* d, int layout, int64_t dim0, int64_t dim1,
                       int64_t dim2, uint8_t* keep);

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
/* with embedding dropout: out = drop_wte(wte[ids]) + drop_wpe(wpe[s]).  The wte mask is elementwise over the [B*S][d]
 * rows (wte->row0 = global row of ids[0][0]); the wpe mask is elementwise over [S][d] (wpe->row0 = 0), one mask shared
 * by every sequence.  bwd: dwte[ids] += dx * keep_wte * scale,  dwpe[s] += keep_wpe[s] * scale * sum_b dx[b,s]. */
int db200_embed_fwd_ex(db200_stream_t stream, const int32_t* ids, const void* wte_bf16, const void* wpe_bf16,
                       void* out_bf16, int B, int S, int d, int V, const db200_dropout* wte_drop,
                       const db200_dropout* wpe_drop);
int db200_embed_bwd_ex(db200_stream_t stream, const int32_t* ids, const void* dx_bf16, float* dwte, float* dwpe, int B,
                       int S, int d, int V, void* workspace, int64_t workspace_bytes, const db200_dropout* wte_drop,
                       const db200_dropout* wpe_drop);
/* same, with every dx element multiplied by alpha in fp32 (rounded on its own) before it is summed: the embedding
 * gradient shrink of the `stable` option, tokens * alpha + tokens.detach() * (1 - alpha), whose forward is
 * unchanged. */
int db200_embed_bwd_scaled(db200_stream_t stream, const int32_t* ids, const void* dx_bf16, float* dwte, float* dwpe,
                           int B, int S, int d, int V, void* workspace, int64_t workspace_bytes,
                           const db200_dropout* wte_drop_or_null, const db200_dropout* wpe_drop_or_null, float alpha);

/* T0 token assembly: tokens[b] = concat(text_ids[b], image_idx[b] + image_offset).  Replaces tf.concat at
 * src/model_fns.py:117-122 (image_offset = text_vocab_size). */
int db200_assemble_tokens(db200_stream_t stream, const int32_t* text_ids, const int32_t* image_idx, int32_t* tokens,
                          int B, int text_len, int image_len, int image_offset);
/* with caption dropout (the training half of classifier-free guidance): every text position of row b becomes pad_id
 * when sequence caption_drop->row0 + b is dropped (D0, site DB200_SITE_CAPTION); image positions are untouched.  NULL
 * or threshold 0 runs db200_assemble_tokens.  pad_id < 0 or row0 < 0 -> DB200_E_INVALID. */
int db200_assemble_tokens_ex(db200_stream_t stream, const int32_t* text_ids, const int32_t* image_idx, int32_t* tokens,
                             int B, int text_len, int image_len, int image_offset, int32_t pad_id,
                             const db200_dropout* caption_drop);
/* with per-position padding (the DALL-E paper's separate padding token for each text position): text position t of
 * row b becomes pad_base + t when its caption id equals pad_id or when the row's caption is dropped (caption_drop as in
 * _ex; NULL or threshold 0: no dropout); other caption ids pass through and image positions are as above.  image_len
 * may be 0 (captions alone, image_idx NULL).  pad_id < 0, pad_base < 0 or row0 < 0 -> DB200_E_INVALID. */
int db200_assemble_tokens_pp(db200_stream_t stream, const int32_t* text_ids, const int32_t* image_idx, int32_t* tokens,
                             int B, int text_len, int image_len, int image_offset, int32_t pad_id, int32_t pad_base,
                             const db200_dropout* caption_drop);

/* Row / column image positions (the DALL-E paper's input embedding).  The image tokens form a grid_w x grid_w grid.
 *   pos_compose: pos bf16 [text_len + grid_w^2][d] from wpe [text_len][d], image_row / image_col [grid_w][d] (bf16):
 *                pos[p] = wpe[p] for p < text_len, pos[text_len + r grid_w + c] = bf16_rn(float(image_row[r]) +
 *                float(image_col[c])).  The embedding kernels read pos where they read an absolute wpe.
 *   pos_fold:    its transpose on fp32 gradients, dpos [text_len + grid_w^2][d]: dwpe[p] += dpos[p],
 *                dimage_row[r] += sum_c dpos[text_len + r grid_w + c] (c ascending), dimage_col[c] += sum_r (r
 *                ascending).  Each sum is formed in fp32 in that order and added once: bit-reproducible.
 * d % 8 == 0, 16-byte aligned pointers (wpe / dwpe may be NULL when text_len == 0). */
int db200_pos_compose(db200_stream_t stream, const void* wpe_bf16, const void* image_row_bf16,
                      const void* image_col_bf16, void* pos_bf16, int text_len, int grid_w, int d);
int db200_pos_fold(db200_stream_t stream, const float* dpos, float* dwpe, float* dimage_row, float* dimage_col,
                   int text_len, int grid_w, int d);

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
/* sandwich LayerNorm (CogView's Sandwich-LN): the branch output o is normalised and added to the residual stream x,
 *     y = bf16(x + (o - mean) * rstd * g + b)            (fp32, one rounding; the normalised o is never rounded alone)
 * mean / rstd of o are computed by the same instructions as db200_layernorm_fwd's, so they are bit-identical to it on
 * the same o.  Same d as db200_layernorm_fwd, any rows > 0.  Backward: db200_layernorm_bwd(_dropout) on o with
 * dres = NULL (the residual's gradient is dy itself). */
int db200_layernorm_residual_fwd(db200_stream_t stream, const void* o_bf16, const void* x_res_bf16, const float* g,
                                 const float* b, void* y_bf16, float* mean, float* rstd, int rows, int d, float eps);
/* backward of LayerNorm whose input x = r + dropout(branch): also writes dxm = dx * keep * scale (the gradient of the
 * branch output before its residual dropout, elementwise mask of `drop` over [rows][d]) and dxsum[c] += sum_rows dxm */
int db200_layernorm_bwd_dropout(db200_stream_t stream, const void* dy_bf16, const void* x_bf16, const float* g,
                                const float* mean, const float* rstd, const void* dres_bf16_or_null, void* dx_bf16,
                                void* dxm_bf16, float* dg, float* db, float* dxsum_or_null, int rows, int d,
                                const db200_dropout* drop, void* workspace, int64_t workspace_bytes);
/* LayerScale (DALLE-pytorch's LayerScale around every branch): the branch output o is scaled per channel by s before
 * the residual add,
 *     y = bf16(x + s[c] * o)                               (fp32, one rounding)
 * any rows > 0, d % 8 == 0, 16-byte aligned operands. */
int db200_layer_scale_residual_fwd(db200_stream_t stream, const void* o_bf16, const void* x_res_bf16, const float* s,
                                   void* y_bf16, int rows, int d);
/* LayerScale on a sandwich LayerNorm's output:
 *     y = bf16(x + s[c] * ((o - mean) * rstd * g + b))       (fp32, one rounding)
 * with mean / rstd of o from the same instructions as db200_layernorm_fwd's.  Same d as db200_layernorm_fwd. */
int db200_layernorm_scale_residual_fwd(db200_stream_t stream, const void* o_bf16, const void* x_res_bf16,
                                       const float* g, const float* b, const float* s, void* y_bf16, float* mean,
                                       float* rstd, int rows, int d, float eps);
/* LayerScale backward from the residual gradient dy and the branch value v the scale multiplied:
 *     dv[r][c]  = bf16(s[c] * dy[r][c] * keep * scale)     (keep * scale: the mask of `drop`, NULL or inactive: 1)
 *     ds[c]    += sum_r dy[r][c] * v[r][c]                 (fp32)
 *     db[c]    += sum_r dv[r][c]                           (the stored bf16 values; db may be NULL)
 * v is the bf16 branch output, or with g != NULL the sandwich LayerNorm output recomputed in fp32 from the stored o,
 * v = (o - mean[r]) * rstd[r] * g[c] + b[c] (b, mean and rstd then required; `drop` must be NULL or inactive, the
 * LayerNorm backward applies it).  Sums go through per-block partial rows of the workspace, added in a fixed order:
 * the result is bit-reproducible.  d % 256 == 0. */
int db200_layer_scale_bwd(db200_stream_t stream, const void* dy_bf16, const void* v_bf16, const float* s,
                          const float* g_or_null, const float* b_or_null, const float* mean_or_null,
                          const float* rstd_or_null, void* dv_bf16, float* ds, float* db_or_null,
                          const db200_dropout* drop_or_null, int rows, int d, void* workspace,
                          int64_t workspace_bytes);
int64_t db200_layer_scale_bwd_workspace_bytes(int rows, int d);
/* DivideMax before a LayerNorm (the `stable` option's final LayerNorm): per row m = max_c x[c] over the bf16 values,
 * u = x / m in fp32 (IEEE division, never rounded to bf16), y = bf16((u - mean) * rstd * g + b) with mean / rstd of u.
 * Writes y, mean, rstd and m (fp32 [rows]).  m = 0 gives the non-finite values of the division.  Same d as
 * db200_layernorm_fwd, any rows > 0. */
int db200_layernorm_divmax_fwd(db200_stream_t stream, const void* x_bf16, const float* g, const float* b, void* y_bf16,
                               float* mean, float* rstd, float* m, int rows, int d, float eps);
/* its backward with m held constant: dx = LN'(u)^T dy / m (+ dres), dg / db / dxsum as db200_layernorm_bwd_ex; with an
 * active `drop` also dxm = dx * keep * scale and dxsum sums dxm, as db200_layernorm_bwd_dropout.  Workspace:
 * db200_layernorm_bwd_workspace_bytes(rows, d). */
int db200_layernorm_divmax_bwd(db200_stream_t stream, const void* dy_bf16, const void* x_bf16, const float* g,
                               const float* mean, const float* rstd, const float* m, const void* dres_bf16_or_null,
                               void* dx_bf16, void* dxm_bf16_or_null, float* dg, float* db, float* dxsum_or_null,
                               int rows, int d, const db200_dropout* drop_or_null, void* workspace,
                               int64_t workspace_bytes);

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
/* residual dropout in the STORE epilogue: D = residual + keep * scale * act(alpha*acc + bias), mask elementwise over
 * [M][N] (needs N % 8 == 0).  Other epilogues take no dropout. */
int db200_gemm_bf16_ex(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda, const void* B, int b_mn_major,
                       int64_t ldb, void* D, int64_t ldd, int M, int N, int K, const db200_gemm_epilogue* epi,
                       const db200_dropout* dropout);
/* Weighted cross-entropy (extension; the reference has no equivalent).  Row m of the vocabulary product is a text row
 * iff m mod period < text_rows, else an image row; it carries the coefficient a = a_text or a_image and the z-loss
 * z_loss * lse[m]^2 (mtf's z_loss).  The loss is sum_m a * (lse[m] - logit[m][label[m]] + z_loss * lse[m]^2).
 * period > 0, 0 <= text_rows <= period, a_text, a_image, z_loss finite and >= 0; otherwise DB200_E_INVALID. */
typedef struct db200_ce_weights {
  int32_t period;     /* rows per sequence (S)                                                     */
  int32_t text_rows;  /* rows per sequence whose target is a text token (text_seq_len - 1)        */
  float a_text;       /* coefficient of a text row's loss                                         */
  float a_image;      /* coefficient of an image row's loss (targets: image tokens and EOS)       */
  float z_loss;       /* z >= 0                                                                   */
} db200_ce_weights;
/* weighted CE_GRAD: D(bf16) = a * ((1 + 2 z lse[m]) exp(acc+bias - lse[m]) - [n == label[m]]), 0 for n >= n_valid;
 * epi->mode must be DB200_EPI_CE_GRAD (epi->alpha is not read), A k-major (DB200_E_UNSUPPORTED otherwise) and B of
 * either major (mn-major: an untied [d][Vpad] projection; k-major: a tied [Vpad][d] embedding).  A row with a = 0
 * gets exact zeros; colsum / workspace as for CE_GRAD. */
int db200_gemm_bf16_ce_weighted(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda, const void* B,
                                int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M, int N, int K,
                                const db200_gemm_epilogue* epi, const db200_ce_weights* w);
/* GELU MLP (extension; the reference's DALLE(activation_fn=...) hook, src/dalle_mtf/models.py:146,177-179,320).
 * mtf's tanh GELU, gelu(x) = x sigma(2u) with u = sqrt(2/pi) (x + 0.044715 x^3), evaluated in fp32.
 * Forward store (the W1 product): z = bf16(alpha*acc + bias[n]); D(bf16) = bf16(gelu(z)); z is also written to
 *   z[M][ldz] (bf16) when z != NULL (training keeps it for backward; inference passes NULL).  epi->mode must be
 *   DB200_EPI_STORE with out_f32 = 0, relu = 0 and no residual; A k-major and B mn-major (DB200_E_UNSUPPORTED
 *   otherwise); N, ldd and ldz multiples of 8 and z 16-byte aligned (DB200_E_ALIGN).
 * Backward (the dgrad dH = dbranch W2^T): D(bf16) = bf16(alpha*acc * gelu'(aux[m,n])) with aux = the stored z;
 *   epi->mode must be DB200_EPI_RELU_BWD (aux, colsum and workspace exactly as for RELU_BWD, so
 *   db200_gemm_workspace_bytes sizes its column-sum workspace); A and B k-major.
 * Finite z gives finite h and gelu'; where sigma is exactly 0 or 1 in fp32, gelu' is exactly 0 or 1.  z = +inf gives
 * h = +inf, z = -inf or NaN gives h = NaN; gelu' of a non-finite z is NaN. */
int db200_gemm_bf16_gelu(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda, const void* B,
                         int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M, int N, int K,
                         const db200_gemm_epilogue* epi, void* z, int64_t ldz);
int db200_gemm_bf16_gelu_bwd(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda, const void* B,
                             int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M, int N, int K,
                             const db200_gemm_epilogue* epi);
/* Gated MLP (extension; DALLE-pytorch's FeedForward: Linear(d, 2*4d), x, gates = chunk(2), x * act(gates)).  N is
 * the width of h (4d); z = [zv | zg] is [M][2N], value columns first.  act: DB200_ACT_RELU (ReGLU) or DB200_ACT_GELU
 * (GEGLU, mtf's tanh GELU evaluated as in db200_gemm_bf16_gelu).
 * Forward store (the W1 product, B = the [K][2N] weight, mn-major, ldb >= 2N): zv = bf16(alpha*acc + bias[n]) over
 *   columns n < N and zg = bf16(alpha*acc + bias[N + n]) over columns N + n; a = bf16(act(zg)) with ReLU's
 *   zg > 0 ? zg : 0 (NaN and -0 give +0); D(bf16) [M][N] = bf16(zv * a); z [M][ldz] (ldz >= 2N) receives zv | zg
 *   when z != NULL.  bias (when given) has 2N entries.  epi->mode must be DB200_EPI_STORE with out_f32 = 0,
 *   relu = 0 and no residual; A k-major and B mn-major (DB200_E_UNSUPPORTED otherwise); N a multiple of 64.
 * Backward (the dgrad dh = dbranch W2^T, A and B k-major, N = the dh width): epi->mode must be DB200_EPI_RELU_BWD
 *   with aux = the stored z (ldaux >= 2N); dh = alpha*acc in fp32, and D(bf16) [M][ldd >= 2N] receives
 *   dzv = bf16(dh * a) in columns n and dzg = bf16((dh * act'(zg)) * zv) in columns N + n, multiplied in that
 *   order, with ReGLU's dh * act'(zg) = zg > 0 ? dh : 0 (the RELU_BWD mask) and GEGLU's dh * gelu'(zg).  colsum (bias gradient, 2N entries) gets the column sums of D as for
 *   RELU_BWD; its workspace is db200_gemm_workspace_bytes(M, 2N, K, epi). */
enum { DB200_ACT_RELU = 0, DB200_ACT_GELU = 1 };
int db200_gemm_bf16_glu(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda, const void* B,
                        int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M, int N, int K,
                        const db200_gemm_epilogue* epi, int act, void* z, int64_t ldz);
int db200_gemm_bf16_glu_bwd(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda, const void* B,
                            int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M, int N, int K,
                            const db200_gemm_epilogue* epi, int act);
/* number of N tiles the CE_STATS epilogue writes per row for a given N (host helper for sizing part_max/part_sum) */
int db200_gemm_ce_tiles(int N);
/* epi->workspace size for this product: split-K slices (ATOMIC) or fused column sums (CE_GRAD / RELU_BWD, which includes
 * the GELU backward, with colsum) */
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
/* weighted finish (db200_ce_weights above): lse[m] as ce_finish; loss_rows[m] = lse[m] - label_logit[m] + z lse[m]^2;
 * sums[0..3] += { sum_m a_m loss_rows[m],  sum over text rows of (lse - label_logit),  the same over image rows,
 * sum_m z lse[m]^2 }.  Per-block partials added in block order: bit-reproducible. */
int db200_ce_finish_weighted(db200_stream_t stream, const float* part_max, const float* part_sum,
                             const float* label_logit, float* lse, float* loss_rows, float* sums, int M, int n_tiles,
                             const db200_ce_weights* w, void* workspace, int64_t workspace_bytes);
int64_t db200_ce_finish_weighted_workspace_bytes(int M);

/* Modality logits mask (extension; DALLE-pytorch's logits_mask).  Row p of each S-row sequence is a text row iff
 * p < text_rows (text_seq_len - 1: its target is a text token) and normalises over vocabulary ids [0, image_offset);
 * the others are image rows (image codes and EOS) and normalise over [image_offset, V).  The vocabulary products run on
 * each class as one contiguous block of rows, the image block over the columns [c0, c0 + round_up(V - c0, 8)) with
 * c0 = image_offset rounded down to a multiple of 8 (a 16-byte aligned TMA base).
 *   partition: hf bf16 [B*S][d] -> hf_text [B*text_rows][d] (rows b*S + p, p < text_rows, in order) and hf_image
 *              [B*(S-text_rows)][d] (the other rows, in order); labels [B*S] -> labels_text (unchanged) and
 *              labels_image (label - c0); bias_image [round_up(V - c0, 8)] = -inf on [c0, image_offset), bias[c] on
 *              [image_offset, V), 0 past V (the -inf columns drop out of every CE epilogue's max, sum and gradient).
 *   scatter:   its inverse on row data: dx bf16 [B*S][d] from dx_text / dx_image and loss_rows [B*S] from loss_text /
 *              loss_image; either triple may be skipped by passing dx (resp. loss_rows) NULL.
 * 0 <= text_rows < S; with text_rows == 0 the text pointers may be NULL.  d % 8 == 0, bf16 pointers 16-byte aligned;
 * 0 <= c0 <= image_offset < V, c0 % 8 == 0.  Row indices are 64-bit; grids are sized from the usable SMs. */
int db200_logits_mask_partition(db200_stream_t stream, const void* hf_bf16, const int32_t* labels, const float* bias,
                                void* hf_text_bf16, void* hf_image_bf16, int32_t* labels_text, int32_t* labels_image,
                                float* bias_image, int B, int S, int text_rows, int d, int c0, int image_offset, int V);
int db200_logits_mask_scatter(db200_stream_t stream, const void* dx_text_bf16, const void* dx_image_bf16,
                              void* dx_bf16, const float* loss_text, const float* loss_image, float* loss_rows, int B,
                              int S, int text_rows, int d);

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
/* attention dropout on the normalised weights before the PV product (attention layout of `drop`; drop->row0 = global
 * index of sequence 0).  lse is that of the undropped weights; out is the dropped output, which backward reads. */
int db200_attn_causal_fwd_ex(db200_stream_t stream, const void* qkv_bf16, void* out_bf16, float* lse, int B, int S,
                             int H, int dh, float scale, const db200_dropout* drop);
int db200_attn_causal_bwd_ex(db200_stream_t stream, const void* qkv_bf16, const void* out_bf16, const void* dout_bf16,
                             const float* lse, float* dq_accum, float* delta, void* dqkv_bf16, int B, int S, int H,
                             int dh, float scale, const db200_dropout* drop);
/* Local (sliding-window) attention of the reference's "local" attention type (mtf local_attention_1d with
 * fully_autoregressive=True, src/dalle_mtf/models.py:257-273): query i attends to keys j with i - radius < j <= i.
 * Layouts, workspaces and numerics as db200_attn_causal_fwd / _bwd; radius >= S is causal attention (bit for bit).
 * No dropout: the reference passes no dropout rate to local attention (models.py:270).  radius < 1: DB200_E_INVALID. */
int db200_attn_local_fwd(db200_stream_t stream, const void* qkv_bf16, void* out_bf16, float* lse, int B, int S, int H,
                         int dh, int radius, float scale);
int db200_attn_local_bwd(db200_stream_t stream, const void* qkv_bf16, const void* out_bf16, const void* dout_bf16,
                         const float* lse, float* dq_accum, float* delta, void* dqkv_bf16, int B, int S, int H, int dh,
                         int radius, float scale);
/* Axial attention of DALL-E's image tokens (DALLE-pytorch's "axial_row" / "axial_col"): a text prefix of text_len
 * positions followed by a grid_w x grid_w image, position p >= text_len being the image token at grid row
 * r = (p - text_len) / grid_w, column c = (p - text_len) % grid_w.  A text query i attends causally to keys j <= i.  An
 * image query attends to every text key and to the image keys of its own row at columns <= c (axis 0, row attention)
 * or of its own column at rows <= r (axis 1, column attention).  S <= text_len + grid_w^2 (a prompt prefill may be
 * shorter).  Layouts, workspaces and numerics as db200_attn_causal_fwd / _bwd.  No dropout.  axis not 0 or 1,
 * grid_w < 1, text_len < 0 or S > text_len + grid_w^2: DB200_E_INVALID. */
int db200_attn_axial_fwd(db200_stream_t stream, const void* qkv_bf16, void* out_bf16, float* lse, int B, int S, int H,
                         int dh, int text_len, int grid_w, int axis, float scale);
int db200_attn_axial_bwd(db200_stream_t stream, const void* qkv_bf16, const void* out_bf16, const void* dout_bf16,
                         const float* lse, float* dq_accum, float* delta, void* dqkv_bf16, int B, int S, int H, int dh,
                         int text_len, int grid_w, int axis, float scale);

/* Convolutional attention of DALL-E's image tokens (DALLE-pytorch's SparseConvCausalAttention at dilation 1), over the
 * grid of db200_attn_axial_fwd.  A text query i attends causally to keys j <= i.  The image query at grid row r,
 * column c attends to every text key and to the image keys at rows r' and columns c' with r - kernel < r' <= r and
 * c - kernel < c' <= c: the kernel x kernel window above and to the left of it, itself included (kernel >= grid_w: every
 * image key at rows <= r and columns <= c).  S <= text_len + grid_w^2 (a prompt prefill may be shorter).  Layouts,
 * workspaces and numerics as db200_attn_causal_fwd / _bwd.  No dropout.  kernel < 1, grid_w < 1, text_len < 0 or
 * S > text_len + grid_w^2: DB200_E_INVALID. */
int db200_attn_conv_fwd(db200_stream_t stream, const void* qkv_bf16, void* out_bf16, float* lse, int B, int S, int H,
                        int dh, int text_len, int grid_w, int kernel, float scale);
int db200_attn_conv_bwd(db200_stream_t stream, const void* qkv_bf16, const void* out_bf16, const void* dout_bf16,
                        const float* lse, float* dq_accum, float* delta, void* dqkv_bf16, int B, int S, int H, int dh,
                        int text_len, int grid_w, int kernel, float scale);

/* Block-sparse attention (DeepSpeed's fixed / variable sparsity layouts, DALLE-pytorch's SparseAttention), described
 * at 16-token granularity by a device table of 16-bit tile masks: tile_mask[qt * mask_pitch + kt] (kt <= qt) for the
 * 64 x 64 tile of queries 64 qt .. 64 qt + 63 and keys 64 kt .. 64 kt + 63; bit 4 a + c set means the queries
 * 64 qt + 16 a .. + 15 may see the keys 64 kt + 16 c .. + 15.  Query i attends to key j iff j <= i, j < S and the bit of
 * (i, j) is set; the same mask serves every head and sequence.  The kernels skip the tiles whose mask is 0 and read
 * the rows qt < ceil(S / 64) of the table only, so a prompt prefill (S shorter than the layout's length) passes the
 * full table.  A query that sees no key gets out = 0.  Layouts, workspaces and numerics as db200_attn_causal_fwd /
 * _bwd; with every causal bit set the results are bit for bit db200_attn_causal_fwd / _bwd's.  No dropout.  A NULL tile_mask or mask_pitch < ceil(S / 64): DB200_E_INVALID. */
int db200_attn_block_sparse_fwd(db200_stream_t stream, const void* qkv_bf16, void* out_bf16, float* lse, int B, int S,
                                int H, int dh, const uint16_t* tile_mask, int mask_pitch, float scale);
int db200_attn_block_sparse_bwd(db200_stream_t stream, const void* qkv_bf16, const void* out_bf16,
                                const void* dout_bf16, const float* lse, float* dq_accum, float* delta, void* dqkv_bf16,
                                int B, int S, int H, int dh, const uint16_t* tile_mask, int mask_pitch, float scale);

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
 * K11p  the DALL-E paper's discrete-VAE network (extension, architecture "dalle_paper"; the reference has none): the
 *     pieces its encoder and decoder need beyond K11's convolutions.  NHWC activations, bf16 (act_f32 = 0) or f32
 *     (act_f32 = 1); 64-bit element counts and offsets throughout.
 *   conv7x7_in_fwd:   the encoder's input conv, y = conv7x7(x, w, stride 1, SAME) + bias, x the f32 image [N][H][W][C]
 *                     (1 <= C <= 4), w f32 [7][7][C][Cout], y [N][H][W][Cout] (Cout % 8 == 0; bf16 or f32).
 *                     Precision: the products and sums are f32 FMAs of the f32 image and the f32 kernel (no bf16
 *                     rounding of either operand, 49 C taps in kh, kw, c order); only the stored output is rounded.
 *   conv7x7_in_wgrad: dw [7][7][C][Cout] += sum over pixels of x[p + tap] dy[p], dbias [Cout] += sum dy (dbias may be
 *                     NULL); dy bf16 or f32.  Per-CTA partials go through the workspace and are added in a fixed
 *                     order: bit-reproducible.  The image's own gradient is never needed and has no kernel.
 *   maxpool2x2_fwd:   y[n][i][j][c] = max of x[n][2i + a][2j + b][c] over the window, H and W even.
 *   maxpool2x2_bwd:   dx = dy at the window's FIRST maximum in raster order (0,0), (0,1), (1,0), (1,1) (a later
 *                     element wins only if strictly greater), 0 at the other three; every dx element is written.  The
 *                     arg-max is recomputed from x (no index tensor).  A NaN only wins as the window's first element.
 *   upsample2x_fwd:   y[n][2i + a][2j + b][c] = x[n][i][j][c] (nearest neighbour); x is [N][H][W][C].
 *   upsample2x_bwd:   dx[n][i][j][c] = ((dy(0,0) + dy(0,1)) + dy(1,0)) + dy(1,1), summed in f32, rounded once.
 *   residual_gain:    v = gain * r + id (one f32 FMA; id NULL: gain * r), then v = 0 where mask <= 0 (mask NULL: no
 *                     mask); y = v rounded to the activation type, relu_y = max(y, 0).  Either output may be NULL,
 *                     not both; y may alias r or id.  A residual block's output x + gain (conv_4 + bias) with the
 *                     ReLU its successor reads, the ReLU alone (id NULL, gain 1), the gradient of the gain-scaled
 *                     path (gain dy) and the ReLU's backward (mask = the ReLU's input).
 * Unsupported geometry (odd H or W for the pool, C outside [1, 4] or Cout % 8 != 0 for the 7x7 conv) returns
 * DB200_E_UNSUPPORTED; there is no fallback.
 * ------------------------------------------------------------------------------------------------------------------ */
int db200_conv7x7_in_fwd(db200_stream_t stream, const float* x, const float* w, const float* bias_or_null, void* y,
                         int N, int H, int W, int C, int Cout, int act_f32);
int db200_conv7x7_in_wgrad(db200_stream_t stream, const float* x, const void* dy, float* dw, float* dbias_or_null,
                           int N, int H, int W, int C, int Cout, int act_f32, void* workspace,
                           int64_t workspace_bytes);
int64_t db200_conv7x7_in_wgrad_workspace_bytes(int N, int H, int W, int C, int Cout);
int db200_maxpool2x2_fwd(db200_stream_t stream, const void* x, void* y, int N, int H, int W, int C, int act_f32);
int db200_maxpool2x2_bwd(db200_stream_t stream, const void* x, const void* dy, void* dx, int N, int H, int W, int C,
                         int act_f32);
int db200_upsample2x_fwd(db200_stream_t stream, const void* x, void* y, int N, int H, int W, int C, int act_f32);
int db200_upsample2x_bwd(db200_stream_t stream, const void* dy, void* dx, int N, int H, int W, int C, int act_f32);
int db200_residual_gain(db200_stream_t stream, const void* id_or_null, const void* r, const void* mask_or_null,
                        float gain, void* y_or_null, void* relu_y_or_null, int64_t n, int act_f32);

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
/* ------------------------------------------------------------------------------------------------------------------
 * K14  a taming-transformers VQGAN tokenizer's forward (extension, architecture "vqgan"; DESIGN.md §4): what its
 *      encoder and decoder need beyond K11's convolutions, the GEMM, upsample2x_fwd, split and argmax_rows.  NHWC bf16
 *      activations.  No float atomics; launch geometries depend on HW and C only, so an image's result does not depend
 *      on N (the batch it is computed in).
 *   groupnorm_stats: mean / rstd f32 [N][G] of x bf16 [N][HW][C] over each image's HW x C/G values of group g
 *                    (channels [g C/G, (g + 1) C/G)): per-thread per-channel Welford states over whole pixel rows,
 *                    combined with Chan's pairwise update in a fixed order, first per chunk of pixel rows into the
 *                    workspace, then across chunks in chunk order; rstd = 1 / sqrt(M2 / count + eps) (biased).
 *                    C % 8 == 0, C % G == 0 and C <= 2048, else DB200_E_UNSUPPORTED; x 16-byte aligned.
 *   groupnorm_apply: y = (x - mean) rstd gamma + beta in f32, then swish(v) = v sigmoid(v) when swish != 0, rounded
 *                    once to bf16.  gamma / beta f32 [C]; x, y 16-byte aligned.
 *   attn_noncausal_fwd: one head over each image's S positions: qkv bf16 [B][S][3C] (q | k | v), out bf16 [B][S][C],
 *                    out_i = sum_j softmax_j(scale q_i . k_j) v_j with fp32 scores, the row maximum subtracted and an
 *                    fp32 weighted sum, rounded once.  S % 64 == 0 and S <= 256, C % 64 == 0 and C <= 512, else
 *                    DB200_E_UNSUPPORTED.  One launch for all B images.
 *   attn_noncausal_long_fwd: the same attention and layout over longer sequences on wgmma: C == 512, S % 64 == 0 and
 *                    256 < S <= 4096, B <= 65535, else DB200_E_UNSUPPORTED.  bf16 q, k, v; fp32 scores (each
 *                    query's two 256-channel halves summed in fp32), an fp32 online softmax over 64-key tiles in key
 *                    order, P rounded to bf16 for the fp32-accumulated P v, rounded once.  No atomics: bit-reproducible,
 *                    and an image's output does not depend on B.  qkv / out 16-byte aligned.
 *   gather_rows_split: hi[r] = bf16(table[idx[r] - offset]), lo[r] = bf16(table row - hi) (lo may be NULL); table f32
 *                    [K][D], hi / lo bf16 [rows][D].  A row whose id is outside [offset, offset + K) is all zeros (as
 *                    db200_onehot_rows_f32 gives a zero one-hot row).
 *   clamp_bf16_to_f32: dst[i] = min(max(float(src[i]), lo), hi) (the decoder's output as an f32 image).
 * ------------------------------------------------------------------------------------------------------------------ */
int db200_groupnorm_stats(db200_stream_t stream, const void* x_bf16, float* mean, float* rstd, int N, int HW, int C,
                          int G, float eps, void* workspace, int64_t workspace_bytes);
int64_t db200_groupnorm_stats_workspace_bytes(int N, int HW, int C, int G);
int db200_groupnorm_apply(db200_stream_t stream, const void* x_bf16, const float* mean, const float* rstd,
                          const float* gamma, const float* beta, void* y_bf16, int N, int HW, int C, int G, int swish);
int db200_attn_noncausal_fwd(db200_stream_t stream, const void* qkv_bf16, void* out_bf16, int B, int S, int C,
                             float scale);
int db200_attn_noncausal_long_fwd(db200_stream_t stream, const void* qkv_bf16, void* out_bf16, int B, int S, int C,
                                  float scale);
int db200_gather_rows_split(db200_stream_t stream, const int32_t* idx, const float* table, void* hi_bf16,
                            void* lo_bf16_or_null, int rows, int D, int K, int offset);
int db200_clamp_bf16_to_f32(db200_stream_t stream, const void* src_bf16, float* dst, int64_t n, float lo, float hi);
/* KL(q_r || Uniform(K)) of the encoder logits l_r, q_r = softmax(l_r) (extension: the KL term of the DALL-E paper's
 * ELB, DALLE-pytorch's kl_div_loss_weight; the reference has neither).  All f32 except the int32 histogram.
 *   vae_kl_stats: lse[r] = logsumexp(l_r);  ent[r] = sum_k q_rk (l_rk - lse[r]);  hist[argmax l_r] += 1 (first maximum,
 *                 a row with a NaN counts as code 0);  *kl_accum += scale * sum_r (ent[r] + log K).  One read of the
 *                 logits; per-CTA partials added in CTA order (bit-reproducible); a row with NaN / inf logits may get a
 *                 NaN lse / ent / KL but writes nothing outside its row and a histogram index in [0, K).
 *   gumbel_softmax_bwd_kl: dlogits = y (dy - sum(dy.*y)) / tau + c q (l - lse - ent)   (q recomputed from l and lse)
 * scale and c must be finite. */
int db200_vae_kl_stats(db200_stream_t stream, const float* logits, float* lse, float* ent, int32_t* hist,
                       float* kl_accum, int rows, int K, float scale, void* workspace, int64_t workspace_bytes);
int64_t db200_vae_kl_stats_workspace_bytes(int rows, int K);
int db200_gumbel_softmax_bwd_kl(db200_stream_t stream, const float* y_soft, const float* dy, const float* logits,
                                const float* lse, const float* ent, float* dlogits, int rows, int K, float tau, float c);
/* Logit-Laplace reconstruction loss (extension: the DALL-E paper's dVAE likelihood; the reference has MSE only).  f32,
 * n_pix pixels of Cp packed channels.  stats [n_pix][2 Cp]: mu in channels [0, Cp), ln b in [Cp, 2 Cp).
 * target [n_pix][Cp] in [-1, 1]: y = clamp(0.1 + 0.8 (x + 1) / 2, 0.1, 0.9), t = ln y - ln(1 - y).
 *   recon_out = clamp(2.5 sigmoid(mu) - 1.25, -1, 1)   (always written)
 * With a target (dstats, nll_accum, mse_accum and the workspace then required):
 *   *nll_accum += scale * sum (ln 2 + ln b + ln y + ln(1 - y) + |t - mu| exp(-ln b));
 *   *mse_accum += scale * sum (recon_out - target)^2;
 *   dstats[mu] = -scale sign(t - mu) exp(-ln b) (sign(0) = 0);  dstats[ln b] = scale (1 - |t - mu| exp(-ln b)).
 * target NULL (decoding): only recon_out is written.  Both sums are per-CTA partials added in CTA order
 * (bit-reproducible); a non-finite stat stays in its own element.  scale must be finite. */
int db200_logit_laplace_fwd_bwd(db200_stream_t stream, const float* stats, const float* target_or_null,
                                float* dstats_or_null, float* recon_out, float* nll_accum, float* mse_accum,
                                int64_t n_pix, int Cp, float scale, void* workspace, int64_t workspace_bytes);
int64_t db200_logit_laplace_workspace_bytes(int64_t n_pix, int Cp);
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
/* attn_decode / attn_decode_dev of a local layer (src/dalle_mtf/models.py:257-273): the query of position p attends to
 * keys [max(0, p - radius + 1), p] of the same full-length cache.  radius >= S is attn_decode; radius < 1 is
 * DB200_E_INVALID. */
int db200_attn_decode_local(db200_stream_t stream, const void* qkv_step_bf16, void* k_cache_bf16, void* v_cache_bf16,
                            void* out_bf16, int B, int S, int H, int dh, int pos, int radius, float scale);
int db200_attn_decode_local_dev(db200_stream_t stream, const void* qkv_step_bf16, void* k_cache_bf16,
                                void* v_cache_bf16, void* out_bf16, int B, int S, int H, int dh,
                                const int32_t* pos_dev, int radius, float scale);
/* attn_decode / attn_decode_dev of an axial layer (db200_attn_axial_fwd's geometry): the query of position p attends
 * to the text keys [0, min(p, text_len - 1)] and, when p is the image token at grid row r, column c, to keys
 * text_len + r grid_w + c' for c' <= c (axis 0) or text_len + r' grid_w + c for r' <= r (axis 1).  The device-position
 * variant sizes shared memory for min(S, text_len + grid_w) keys.  Invalid geometry as db200_attn_axial_fwd. */
int db200_attn_decode_axial(db200_stream_t stream, const void* qkv_step_bf16, void* k_cache_bf16, void* v_cache_bf16,
                            void* out_bf16, int B, int S, int H, int dh, int pos, int text_len, int grid_w, int axis,
                            float scale);
int db200_attn_decode_axial_dev(db200_stream_t stream, const void* qkv_step_bf16, void* k_cache_bf16,
                                void* v_cache_bf16, void* out_bf16, int B, int S, int H, int dh,
                                const int32_t* pos_dev, int text_len, int grid_w, int axis, float scale);
/* attn_decode / attn_decode_dev of a convolutional layer (db200_attn_conv_fwd's geometry): the query of position p
 * attends to the text keys [0, min(p, text_len - 1)] and, when p is the image token at grid row r, column c, to the
 * keys text_len + r' grid_w + c' for max(0, r - kernel + 1) <= r' <= r and max(0, c - kernel + 1) <= c' <= c.  The
 * device-position variant sizes shared memory for min(S, text_len + kernel min(kernel, grid_w)) keys.  Invalid
 * geometry as db200_attn_conv_fwd. */
int db200_attn_decode_conv(db200_stream_t stream, const void* qkv_step_bf16, void* k_cache_bf16, void* v_cache_bf16,
                           void* out_bf16, int B, int S, int H, int dh, int pos, int text_len, int grid_w, int kernel,
                           float scale);
int db200_attn_decode_conv_dev(db200_stream_t stream, const void* qkv_step_bf16, void* k_cache_bf16,
                               void* v_cache_bf16, void* out_bf16, int B, int S, int H, int dh,
                               const int32_t* pos_dev, int text_len, int grid_w, int kernel, float scale);
/* attn_decode / attn_decode_dev of a block-sparse layer: the query of position p attends to the keys of the 16-key
 * blocks listed for 16-row block g = p / 16, clipped at p.  `blocks` is a device table of rows of blocks_pitch int32:
 * row g holds a count n_g followed by n_g distinct block indices in ascending order, each <= g (the layout of
 * db200_attn_block_sparse_fwd at 16-token granularity).  A position whose row lists no block gets out = 0.  Shared
 * memory and key counts as db200_attn_decode / _dev.  A NULL table or blocks_pitch < ceil(S / 16) + 1:
 * DB200_E_INVALID. */
int db200_attn_decode_block_sparse(db200_stream_t stream, const void* qkv_step_bf16, void* k_cache_bf16,
                                   void* v_cache_bf16, void* out_bf16, int B, int S, int H, int dh, int pos,
                                   const int32_t* blocks, int blocks_pitch, float scale);
int db200_attn_decode_block_sparse_dev(db200_stream_t stream, const void* qkv_step_bf16, void* k_cache_bf16,
                                       void* v_cache_bf16, void* out_bf16, int B, int S, int H, int dh,
                                       const int32_t* pos_dev, const int32_t* blocks, int blocks_pitch, float scale);
int db200_sample_rows_at(db200_stream_t stream, const float* logits, const float* u_or_null, int32_t* tokens,
                         long long ld_tokens, int rows, long long ld, int lo, int hi, float inv_temp,
                         const int32_t* pos_dev);
int db200_incr_i32(db200_stream_t stream, int32_t* p, int delta);
/* Top-k / nucleus (top-p) filtered sample_rows.  Per row, over x_c = logits[r][lo + c] * inv_temp (c < n = hi - lo):
 *   top-k (top_k >= 1; 0 = off): keep x_c >= the k-th largest x (counting multiplicity; ties at it are all kept, so
 *          more than k ids may survive; k >= n keeps everything);
 *   top-p (0 < top_p <= 1; 1 = off): over the top-k survivors, with w = exp(x - max) and Z = sum w, keep x_c iff the
 *          mass of the survivors strictly greater than x_c is < top_p * Z (independent of how ties are ordered; the
 *          maximum is always kept);
 *   idx[r] = lo + argmax over the kept c of (x_c - log(-log u[r][c])), first index on ties; u NULL = greedy, which
 *          the filter cannot change.  With the filter off the selection is exactly sample_rows'.
 * NaN and -inf are never kept; a row with no finite entry gives lo and a kept count of 0; +inf entries, if any, are
 * the only ones kept.  kept_or_null (int32 [rows]) receives the number of kept ids; the kept set is the top that many
 * x, so the count identifies it.  Results are bit-reproducible (masses are summed in 64-bit fixed point).
 * One CTA holds a row: n <= 51 200, larger n returns DB200_E_UNSUPPORTED.  top_k < 0, top_p NaN / <= 0 / > 1,
 * inv_temp <= 0 and an empty range return DB200_E_INVALID.  The _at variant writes tokens[r * ld_tokens + *pos_dev + 1]
 * like db200_sample_rows_at. */
int db200_sample_rows_filtered(db200_stream_t stream, const float* logits, const float* u_or_null, int32_t* idx,
                               int32_t* kept_or_null, int rows, long long ld, int lo, int hi, float inv_temp,
                               int top_k, float top_p);
int db200_sample_rows_filtered_at(db200_stream_t stream, const float* logits, const float* u_or_null, int32_t* tokens,
                                  long long ld_tokens, int32_t* kept_or_null, int rows, long long ld, int lo, int hi,
                                  float inv_temp, int top_k, float top_p, const int32_t* pos_dev);
/* Classifier-free guidance over `rows` pairs.  logits f32 [2*rows][ld]: rows [0, rows) are conditional (c), rows
 * [rows, 2*rows) unconditional (u).  Pair r samples, with the rules above, from
 *   x_c = g * inv_temp,  g = __fadd_rn(u, __fmul_rn(s, __fsub_rn(c, u)))   (s = guidance_scale; no FMA contraction,
 *                                                                           so a float32 host computation matches)
 * through top-k, then top-p, then the Gumbel-max with noise row r of u_or_null (f32 [rows][hi-lo]; NULL = greedy).
 * A NaN g is never kept or selected.  The draw is written to tokens[r * ld_tokens + col] and
 * tokens[(rows + r) * ld_tokens + col], col = pos_dev ? *pos_dev + 1 : 0, so both rows continue with the same token.
 * top_k == 0 && top_p == 1 runs the unfiltered kernel (kept_or_null must then be NULL), anything else the filtered one
 * (kept_or_null: int32 [rows]).  guidance_scale NaN / inf / < 0, ld_tokens < 1 and the argument errors of
 * db200_sample_rows_filtered return DB200_E_INVALID. */
int db200_sample_rows_guided(db200_stream_t stream, const float* logits, long long ld, const float* u_or_null,
                             int32_t* tokens, long long ld_tokens, int32_t* kept_or_null, int rows, int lo, int hi,
                             float inv_temp, float guidance_scale, int top_k, float top_p,
                             const int32_t* pos_dev_or_null);
/* Caption completion: finishes text column c = pos + 1 of every row of the int32 token matrix tokens [rows][ld_tokens]
 * after a draw has been written into it (run it after any of the samplers above).  For row b, with n_b = lens[b]:
 *   c < n_b              : tokens[b][c] = prefix[b][c]   (the prompt, prefix int32 [rows][ld_prefix] in token form)
 *   else if tokens[b][c - 1] or tokens[b][c] is a padding token : tokens[b][c] = c's pad
 *   else                 : the draw is kept.
 * A padding token is padding_id or, with per-position padding (pad_base >= 0), any id >= text_vocab_size; c's pad is
 * pad_base + c, or padding_id when pad_base < 0.  Integer arithmetic only: the result is exact.  The _at variant reads
 * pos from device memory (graph replay) and leaves the matrix unchanged when c is outside [1, text_len).  A null
 * pointer, rows < 1, ld_tokens or ld_prefix < text_len, padding_id outside [0, text_vocab_size), 0 <= pad_base <
 * text_vocab_size, or (host position) c outside [1, text_len): DB200_E_INVALID. */
int db200_caption_next(db200_stream_t stream, int32_t* tokens, long long ld_tokens, const int32_t* prefix,
                       long long ld_prefix, const int32_t* lens, int rows, int text_len, int text_vocab_size,
                       int padding_id, int pad_base, int pos);
int db200_caption_next_at(db200_stream_t stream, int32_t* tokens, long long ld_tokens, const int32_t* prefix,
                          long long ld_prefix, const int32_t* lens, int rows, int text_len, int text_vocab_size,
                          int padding_id, int pad_base, const int32_t* pos_dev);
/* Prompt prefill hand-off: a whole prompt runs through the training forward kernels at sequence length P, and these
 * copies turn its results into the decoder's state (bandwidth-bound, 16-byte vector accesses).
 *   kv_cache_fill : qkv bf16 [B][P][3][H][dh] (the fused q|k|v GEMM output attn_causal_fwd reads) -> caches bf16
 *                   [B*rep][S_cache][H][dh] (the attn_decode layout): for b < B, p < P, r < rep
 *                   k_cache[b*rep + r][p] = qkv[b][p][1], v_cache[b*rep + r][p] = qkv[b][p][2]; positions >= P are
 *                   not written.  P > S_cache, rep < 1 or a non-positive size -> DB200_E_INVALID; H*dh not a multiple
 *                   of 8 or an unaligned pointer -> DB200_E_ALIGN.
 *   rows_repeat   : dst bf16 [B*rep][d] row b*rep + r = src row b, src rows ld_src elements apart (e.g. the last prompt
 *                   position of a [B][P][d] residual stream: src = x + (P-1)*d, ld_src = P*d).  d and ld_src must be
 *                   multiples of 8 and the pointers 16-byte aligned (DB200_E_ALIGN). */
int db200_kv_cache_fill(db200_stream_t stream, const void* qkv_bf16, void* k_cache_bf16, void* v_cache_bf16, int B,
                        int P, int H, int dh, int S_cache, int rep);
int db200_rows_repeat(db200_stream_t stream, const void* src_bf16, long long ld_src, void* dst_bf16, int B, int d,
                      int rep);

/* Rotary position embeddings (extension; GPT-NeoX's rotate_half layout with partial rotary r = rotary_dim).  qkv is
 * bf16 [rows][3][H][dh], rotated in place: for every q and k head of row t at position p, with h = r / 2 and j < h,
 *   x_j' = bf16(x_j c - x_{j+h} s),  x_{j+h}' = bf16(x_{j+h} c + x_j s),  c = table[p][0][j], s = table[p][1][j],
 * every product and sum rounded separately in fp32 (no FMA contraction).  v and the dims r .. dh-1 are unchanged.
 * table: fp32 [n_pos][2][h], position p's cosines then its sines of p theta_j (theta_j = base^(-2j/r)).
 *   rope_fwd        : p = t mod S; the table holds at least S positions.
 *   rope_bwd        : the transpose rotation (s -> -s) of rope_fwd, applied to the dq and dk columns of dqkv.
 *   rope_decode     : every row at position pos, 0 <= pos < S (the table's, and the cache's, length).
 *   rope_decode_dev : every row at position *pos_dev (graph replay); a position outside [0, S) leaves qkv unchanged.
 * r even with 2 <= r <= dh, rows, S, H, dh > 0 and non-NULL pointers, else DB200_E_INVALID; when h % 8 == 0 and
 * dh % 8 == 0 (16-byte vectors) qkv and the table must be 16-byte aligned (DB200_E_ALIGN). */
int db200_rope_fwd(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S, int H, int dh, int r);
int db200_rope_bwd(db200_stream_t stream, void* dqkv_bf16, const float* table, int rows, int S, int H, int dh, int r);
int db200_rope_decode(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S, int H, int dh, int r,
                      int pos);
int db200_rope_decode_dev(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S, int H, int dh,
                          int r, const int32_t* pos_dev);

/* DALLE-pytorch's rotary embedding (rotary_emb; extension).  qkv is bf16 [rows][3][H][dh], rotated in place: for
 * every q, k AND v head of row t at position p and every pair m < pairs (interleaved dims 2m, 2m+1),
 *   x_2m' = bf16(x_2m c - x_2m+1 s),  x_2m+1' = bf16(x_2m+1 c + x_2m s),  c = table[p][0][m], s = table[p][1][m],
 * every product and sum rounded separately in fp32 (no FMA contraction).  The dims 2 pairs .. dh-1 are unchanged.
 * table: fp32 [S][2][pairs], position p's cosines then its sines (the engine's rotary_emb_table: pairs = 3 (dh / 3 / 2),
 * text, image-row and image-column angles).  The position logic is rope_*'s:
 *   rope_emb_fwd        : p = t mod S.
 *   rope_emb_bwd        : the transpose rotation (s -> -s), applied to the dq, dk and dv columns of dqkv.
 *   rope_emb_decode     : every row at position pos, 0 <= pos < S.
 *   rope_emb_decode_dev : every row at position *pos_dev (graph replay); a position outside [0, S) leaves qkv unchanged.
 * 1 <= pairs <= dh / 2, dh even, rows, S, H > 0 and non-NULL pointers, else DB200_E_INVALID; qkv must be 16-byte
 * aligned when dh % 8 == 0 (16-byte vectors of 4 pairs) and 4-byte aligned otherwise, the table 4-byte aligned
 * (DB200_E_ALIGN). */
int db200_rope_emb_fwd(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S, int H, int dh,
                       int pairs);
int db200_rope_emb_bwd(db200_stream_t stream, void* dqkv_bf16, const float* table, int rows, int S, int H, int dh,
                       int pairs);
int db200_rope_emb_decode(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S, int H, int dh,
                          int pairs, int pos);
int db200_rope_emb_decode_dev(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S, int H,
                              int dh, int pairs, const int32_t* pos_dev);

/* Token shift (extension; DALLE-pytorch's PreShiftToken) on a bf16 [rows][d] LayerNorm output y, c = d / 4.  Position
 * p < text_len (TL) is a text token, p >= TL the image token u = p - TL at grid row u / grid_w, column u % grid_w.
 * shift(y)[p] keeps y[p][2c, d) and replaces
 *   text p       : [0, 2c) by y[p-1][0, 2c)                                 (zeros at p = 0)
 *   image (r, k) : [0, c) by y[p - grid_w][0, c) if r >= 1, [c, 2c) by y[p-1][c, 2c) if k >= 1, zeros otherwise
 * Pure copies (16-byte vectors, 64-bit offsets): exact.
 *   shift_tokens_fwd        : out = shift(y), row t at position t mod S (out of place).
 *   shift_tokens_bwd        : dy = shift^T(dout): text p gets dout[p+1][0, 2c) if p + 1 < TL; image (r, k) gets
 *                             dout[p + grid_w][0, c) if r + 1 < grid_w and dout[p+1][c, 2c) if k + 1 < grid_w
 *                             (sources at positions >= S excluded); [2c, d) is copied.
 *   shift_tokens_decode     : one decoding step at position pos, in place on y [rows][d] with the cache bf16
 *                             [rows][S][d/2]: cache[b][pos] = y[b][0, 2c), then y[b][0, 2c) = the shifted chunks read
 *                             from cache[b][pos-1] / cache[b][pos-grid_w] (or zeros).  0 <= pos < S.
 *   shift_tokens_decode_dev : the same at position *pos_dev (graph replay); a position outside [0, S) changes nothing.
 *   shift_cache_fill        : prefill hand-off, y bf16 [B][P][d] -> cache [B*rep][S_cache][d/2]: cache[b*rep + r][p] =
 *                             y[b][p][0, 2c) for p < P, r < rep (kv_cache_fill's replica order).
 * rows, S, d, grid_w > 0, text_len >= 0, S <= text_len + grid_w^2, d % 32 == 0, non-NULL and non-overlapping buffers,
 * else DB200_E_INVALID; pointers not 16-byte aligned -> DB200_E_ALIGN. */
int db200_shift_tokens_fwd(db200_stream_t stream, const void* y_bf16, void* out_bf16, int rows, int S, int d,
                           int text_len, int grid_w);
int db200_shift_tokens_bwd(db200_stream_t stream, const void* dout_bf16, void* dy_bf16, int rows, int S, int d,
                           int text_len, int grid_w);
int db200_shift_tokens_decode(db200_stream_t stream, void* y_bf16, void* cache_bf16, int rows, int S, int d,
                              int text_len, int grid_w, int pos);
int db200_shift_tokens_decode_dev(db200_stream_t stream, void* y_bf16, void* cache_bf16, int rows, int S, int d,
                                  int text_len, int grid_w, const int32_t* pos_dev);
int db200_shift_cache_fill(db200_stream_t stream, const void* y_bf16, void* cache_bf16, int B, int P, int d,
                           int S_cache, int rep);

/* gMLP token mixing (extension; the spatial gating unit of "Pay Attention to MLPs", DALLE-pytorch's attention type
 * 'mlp').  B sequences of n positions are rows b n .. b n + n - 1 of bf16 [B n][C] activations; W is the bf16
 * [n][ldw] top-left block of the layer's causal mixing weight, whose strict upper triangle is zero.  Sums are fp32
 * over wgmma (bf16 products, fp32 accumulation); one launch per call.
 *   sgu_mix_fwd   : acc[b][i][c] = sum_{j <= i} W[i][j] gn[b n + j][c]; m = acc + c_sgu[i] (fp32);
 *                   h = bf16(m res[b n + i][c]) (res: pitch ldres); mixed (or NULL) = bf16(m).  Any n >= 1.
 *   sgu_mix_dgrad : dgn[b n + j][c] = bf16(sum_{i >= j} W[i][j] dmixed[b n + i][c]).  n % 64 == 0.
 *   sgu_mix_wgrad : dW[i][j] (fp32, pitch ldw) += sum_b sum_c dmixed[b n + i][c] gn[b n + j][c] for j <= i only;
 *                   elements with j > i are never written.  n % 64 == 0.
 *   sgu_bwd       : dmixed = bf16(dh res); du_res (pitch ldu) = bf16(dh mixed gelu'(z_res)) with mtf's tanh GELU;
 *                   dc[i] += sum over b, then c, of dmixed[b n + i][c] (fixed order).
 *   sgu_gate_bwd  : du_gate[t][c] (pitch ldu) = bf16(dgate[t][c] gelu'(z_gate[t][c])), dgate contiguous [rows][C].
 *   sgu_decode    : one decoding step at position pos for every row r, cache bf16 [rows][S][C]: cache[r][pos] = gn[r],
 *                   then h[r][c] = bf16((sum_{j <= pos} W[pos][j] cache[r][j][c] + c_sgu[pos]) res[r][c]), the sum in
 *                   fp32 in j order.  0 <= pos < S <= 12288.
 *   sgu_decode_dev: the same at position *pos_dev (graph replay); a position outside [0, S) changes nothing.
 *   sgu_cache_fill: prefill hand-off, gn bf16 [B P][C] -> cache [B rep][S_cache][C]: cache[b rep + r][p] = gn[b P + p].
 * C % 64 == 0 (mixing products) or even (elementwise, C % 8 == 0 for the cache fill), ldw >= n, ldw % 8 == 0 and
 * non-NULL pointers, else DB200_E_INVALID / DB200_E_ALIGN. */
int db200_sgu_mix_fwd(db200_stream_t stream, const void* w_bf16, int64_t ldw, const void* gn_bf16, const void* res_bf16,
                      int64_t ldres, const float* c, void* h_bf16, void* mixed_bf16, int B, int n, int C);
int db200_sgu_mix_dgrad(db200_stream_t stream, const void* w_bf16, int64_t ldw, const void* dmixed_bf16,
                        void* dgn_bf16, int B, int n, int C);
int db200_sgu_mix_wgrad(db200_stream_t stream, const void* dmixed_bf16, const void* gn_bf16, float* dw, int64_t ldw,
                        int B, int n, int C);
int db200_sgu_bwd(db200_stream_t stream, const void* dh_bf16, const void* mixed_bf16, const void* res_bf16,
                  int64_t ldres, const void* z_bf16, int64_t ldz, void* dmixed_bf16, void* du_bf16, int64_t ldu,
                  float* dc, int B, int n, int C);
int db200_sgu_gate_bwd(db200_stream_t stream, const void* dgate_bf16, const void* z_bf16, int64_t ldz, void* du_bf16,
                       int64_t ldu, int rows, int C);
int db200_sgu_decode(db200_stream_t stream, const void* gn_bf16, const void* res_bf16, int64_t ldres,
                     const void* w_bf16, int64_t ldw, const float* c, void* cache_bf16, void* h_bf16, int rows, int S,
                     int C, int pos);
int db200_sgu_decode_dev(db200_stream_t stream, const void* gn_bf16, const void* res_bf16, int64_t ldres,
                         const void* w_bf16, int64_t ldw, const float* c, void* cache_bf16, void* h_bf16, int rows,
                         int S, int C, const int32_t* pos_dev);
int db200_sgu_cache_fill(db200_stream_t stream, const void* gn_bf16, void* cache_bf16, int B, int P, int C,
                         int S_cache, int rep);

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
