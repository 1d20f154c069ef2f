// K4 — causal flash attention, forward and backward: the C-ABI entry points and the row-wise delta pre-pass.
//
// Replaces mtf_transformer.attention.attention + the [S,S] additive -1e10 mask the reference materialises
// (src/dalle_mtf/models.py:221-227, 287-299).  Logits are fp32 (wgmma accumulators), softmax is fp32, P is rounded to
// bf16 for the PV product (what mtf does when it casts the weights to v's dtype), nothing of size S x S reaches HBM.
// `scale` multiplies q.k (reference: 1.0 — mtf folds 1/sqrt(dh) into the q initialiser).
//
// Layout: qkv bf16 [B][S][3][H][dh] (the fused q|k|v projection output), out / dout bf16 [B][S][H][dh],
//         lse f32 [B][H][S] (natural log of sum exp(scale*s)), dqkv like qkv.
//
// The kernels are in attn_fa.cu (one warpgroup per 64 rows, P / dS handed to the next wgmma in registers); this file
// validates the arguments, runs delta = rowsum(dO * O) and launches them.
#include "common.cuh"
#include "ptx.cuh"

namespace db200 {

int attn_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, int dh,
                    float scale, const db200_dropout* drop);
int attn_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                       void* dqkv, int B, int S, int H, int dh, float scale, const db200_dropout* drop);
int attn_local_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, int dh,
                          int radius, float scale);
int attn_local_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                          void* dqkv, int B, int S, int H, int dh, int radius, float scale);
int attn_axial_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, int dh,
                          int text_len, int grid_w, int axis, float scale);
int attn_axial_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                          void* dqkv, int B, int S, int H, int dh, int text_len, int grid_w, int axis, float scale);
int attn_conv_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, int dh,
                         int text_len, int grid_w, int kernel, float scale);
int attn_conv_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                         void* dqkv, int B, int S, int H, int dh, int text_len, int grid_w, int kernel, float scale);
int attn_block_sparse_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H,
                                 int dh, const uint16_t* mask, int pitch, float scale);
int attn_block_sparse_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse,
                                 const float* delta, void* dqkv, int B, int S, int H, int dh, const uint16_t* mask,
                                 int pitch, float scale);

// ------------------------------------------------------------------------------------------------------------------
// backward: delta = rowsum(dO * O)
// ------------------------------------------------------------------------------------------------------------------
// DH / 8 lanes share one (b, s, h) row (16-byte loads), so a warp covers 32 * 8 / DH consecutive rows = 512 contiguous
// bytes of O and of dO per instruction: HBM-bound (the thread-per-2-elements version was issue-bound at 4x the time).
template <int DH>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const bf16* __restrict__ o, const bf16* __restrict__ dout, float* __restrict__ delta, int B, int S,
                  int H) {
  constexpr int LPR = DH / 8;  // lanes per row
  const long long rows = (long long)B * S * H;
  const long long gt = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long row = gt / LPR;
  const int sub = (int)(gt % LPR);
  float acc = 0.f;
  if (row < rows) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(o + row * DH) + sub);
    const uint4 d = __ldg(reinterpret_cast<const uint4*>(dout + row * DH) + sub);
    const uint32_t av[4] = {a.x, a.y, a.z, a.w}, dv[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 x = unpack_bf16x2(av[i]), y = unpack_bf16x2(dv[i]);
      acc = fmaf(x.x, y.x, acc);
      acc = fmaf(x.y, y.y, acc);
    }
  }
#pragma unroll
  for (int ofs = LPR / 2; ofs > 0; ofs >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, ofs);
  if (row < rows && sub == 0) {
    const int hh = (int)(row % H);
    const long long bs = row / H;
    delta[((long long)(bs / S) * H + hh) * S + (bs % S)] = acc;
  }
}


}  // namespace db200

using namespace db200;

static int attn_delta(cudaStream_t stream, const void* out, const void* dout, float* delta, int B, int S, int H,
                      int dh) {
  const long long threads = (long long)B * S * H * (dh / 8);
  const unsigned blocks = (unsigned)((threads + 255) / 256);
  if (dh == 128)
    attn_delta_kernel<128><<<blocks, 256, 0, stream>>>((const bf16*)out, (const bf16*)dout, delta, B, S, H);
  else
    attn_delta_kernel<64><<<blocks, 256, 0, stream>>>((const bf16*)out, (const bf16*)dout, delta, B, S, H);
  return check_launch("attn_delta_kernel");
}

extern "C" int db200_attn_causal_fwd_ex(db200_stream_t stream_, const void* qkv, void* out, float* lse, int B,
                                        int S, int H, int dh, float scale, const db200_dropout* drop) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && S > 0 && H > 0, DB200_E_INVALID, "attn_fwd: B,S,H must be positive");
  DB200_REQUIRE(qkv && out && lse && aligned16(qkv) && aligned16(out), DB200_E_ALIGN,
                "attn_fwd: NULL or unaligned pointer");
  DB200_REQUIRE(scale > 0.f, DB200_E_INVALID, "attn_fwd: scale must be > 0");
  if (dh != 64 && dh != 128) return set_error(DB200_E_UNSUPPORTED, "attn: head_dim %d not in {64,128}", dh);
  return attn_fwd_launch(stream, qkv, out, lse, B, S, H, dh, scale, drop);
}

extern "C" int db200_attn_causal_fwd(db200_stream_t stream_, const void* qkv, void* out, float* lse, int B, int S,
                                     int H, int dh, float scale) {
  return db200_attn_causal_fwd_ex(stream_, qkv, out, lse, B, S, H, dh, scale, nullptr);
}

extern "C" int db200_attn_causal_bwd_ex(db200_stream_t stream_, const void* qkv, const void* out, const void* dout,
                                        const float* lse, float* dq_accum, float* delta, void* dqkv, int B, int S,
                                        int H, int dh, float scale, const db200_dropout* drop) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  (void)dq_accum;  // kept in the ABI for an atomics-based variant; the two-kernel scheme does not need it
  DB200_REQUIRE(B > 0 && S > 0 && H > 0, DB200_E_INVALID, "attn_bwd: B,S,H must be positive");
  DB200_REQUIRE(qkv && out && dout && lse && delta && dqkv && aligned16(qkv) && aligned16(out) && aligned16(dout) &&
                    aligned16(dqkv),
                DB200_E_ALIGN, "attn_bwd: NULL or unaligned pointer");
  DB200_REQUIRE(scale > 0.f, DB200_E_INVALID, "attn_bwd: scale must be > 0");
  DB200_REQUIRE(dh == 64 || dh == 128, DB200_E_UNSUPPORTED, "attn: head_dim %d not in {64,128}", dh);
  const int rc = attn_delta(stream, out, dout, delta, B, S, H, dh);
  if (rc != DB200_OK) return rc;
  // delta = rowsum(dO * O) needs no dropout term: O already is the dropped output
  return attn_bwd_launch(stream, qkv, dout, lse, delta, dqkv, B, S, H, dh, scale, drop);
}

extern "C" int db200_attn_causal_bwd(db200_stream_t stream_, const void* qkv, const void* out, const void* dout,
                                     const float* lse, float* dq_accum, float* delta, void* dqkv, int B, int S, int H,
                                     int dh, float scale) {
  return db200_attn_causal_bwd_ex(stream_, qkv, out, dout, lse, dq_accum, delta, dqkv, B, S, H, dh, scale, nullptr);
}

// ---- local (sliding-window) attention, src/dalle_mtf/models.py:257-273: query i attends to keys (i - radius, i].
// radius >= S is causal attention (same result as db200_attn_causal_*, bit for bit).  No dropout.
extern "C" int db200_attn_local_fwd(db200_stream_t stream_, const void* qkv, void* out, float* lse, int B, int S, int H,
                                    int dh, int radius, float scale) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && S > 0 && H > 0, DB200_E_INVALID, "attn_local_fwd: B,S,H must be positive");
  DB200_REQUIRE(radius >= 1, DB200_E_INVALID, "attn_local_fwd: radius %d < 1", radius);
  DB200_REQUIRE(qkv && out && lse && aligned16(qkv) && aligned16(out), DB200_E_ALIGN,
                "attn_local_fwd: NULL or unaligned pointer");
  DB200_REQUIRE(scale > 0.f, DB200_E_INVALID, "attn_local_fwd: scale must be > 0");
  DB200_REQUIRE(dh == 64 || dh == 128, DB200_E_UNSUPPORTED, "attn: head_dim %d not in {64,128}", dh);
  return attn_local_fwd_launch(stream, qkv, out, lse, B, S, H, dh, radius, scale);
}

extern "C" int db200_attn_local_bwd(db200_stream_t stream_, const void* qkv, const void* out, const void* dout,
                                    const float* lse, float* dq_accum, float* delta, void* dqkv, int B, int S, int H,
                                    int dh, int radius, float scale) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  (void)dq_accum;
  DB200_REQUIRE(B > 0 && S > 0 && H > 0, DB200_E_INVALID, "attn_local_bwd: B,S,H must be positive");
  DB200_REQUIRE(radius >= 1, DB200_E_INVALID, "attn_local_bwd: radius %d < 1", radius);
  DB200_REQUIRE(qkv && out && dout && lse && delta && dqkv && aligned16(qkv) && aligned16(out) && aligned16(dout) &&
                    aligned16(dqkv),
                DB200_E_ALIGN, "attn_local_bwd: NULL or unaligned pointer");
  DB200_REQUIRE(scale > 0.f, DB200_E_INVALID, "attn_local_bwd: scale must be > 0");
  DB200_REQUIRE(dh == 64 || dh == 128, DB200_E_UNSUPPORTED, "attn: head_dim %d not in {64,128}", dh);
  const int rc = attn_delta(stream, out, dout, delta, B, S, H, dh);
  if (rc != DB200_OK) return rc;
  return attn_local_bwd_launch(stream, qkv, dout, lse, delta, dqkv, B, S, H, dh, radius, scale);
}

// ---- axial (row / column) attention of DALL-E image tokens: text queries are causal; an image query at grid row r,
// column c (position text_len + r grid_w + c) sees every text key and the image keys of row r at columns <= c
// (axis 0) or of column c at rows <= r (axis 1).  S <= text_len + grid_w^2 (a prefill may be shorter).  No dropout.
static int axial_args_ok(const char* fn, int S, int text_len, int grid_w, int axis) {
  DB200_REQUIRE(axis == 0 || axis == 1, DB200_E_INVALID, "%s: axis %d not 0 (row) or 1 (column)", fn, axis);
  DB200_REQUIRE(grid_w >= 1 && text_len >= 0, DB200_E_INVALID, "%s: grid_w %d < 1 or text_len %d < 0", fn, grid_w,
                text_len);
  DB200_REQUIRE((long long)S <= (long long)text_len + (long long)grid_w * grid_w, DB200_E_INVALID,
                "%s: S %d exceeds text_len %d + grid_w^2 (%d^2)", fn, S, text_len, grid_w);
  return DB200_OK;
}

extern "C" int db200_attn_axial_fwd(db200_stream_t stream_, const void* qkv, void* out, float* lse, int B, int S, int H,
                                    int dh, int text_len, int grid_w, int axis, float scale) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && S > 0 && H > 0, DB200_E_INVALID, "attn_axial_fwd: B,S,H must be positive");
  const int arc = axial_args_ok("attn_axial_fwd", S, text_len, grid_w, axis);
  if (arc != DB200_OK) return arc;
  DB200_REQUIRE(qkv && out && lse && aligned16(qkv) && aligned16(out), DB200_E_ALIGN,
                "attn_axial_fwd: NULL or unaligned pointer");
  DB200_REQUIRE(scale > 0.f, DB200_E_INVALID, "attn_axial_fwd: scale must be > 0");
  DB200_REQUIRE(dh == 64 || dh == 128, DB200_E_UNSUPPORTED, "attn: head_dim %d not in {64,128}", dh);
  return attn_axial_fwd_launch(stream, qkv, out, lse, B, S, H, dh, text_len, grid_w, axis, scale);
}

extern "C" int db200_attn_axial_bwd(db200_stream_t stream_, const void* qkv, const void* out, const void* dout,
                                    const float* lse, float* dq_accum, float* delta, void* dqkv, int B, int S, int H,
                                    int dh, int text_len, int grid_w, int axis, float scale) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  (void)dq_accum;
  DB200_REQUIRE(B > 0 && S > 0 && H > 0, DB200_E_INVALID, "attn_axial_bwd: B,S,H must be positive");
  const int arc = axial_args_ok("attn_axial_bwd", S, text_len, grid_w, axis);
  if (arc != DB200_OK) return arc;
  DB200_REQUIRE(qkv && out && dout && lse && delta && dqkv && aligned16(qkv) && aligned16(out) && aligned16(dout) &&
                    aligned16(dqkv),
                DB200_E_ALIGN, "attn_axial_bwd: NULL or unaligned pointer");
  DB200_REQUIRE(scale > 0.f, DB200_E_INVALID, "attn_axial_bwd: scale must be > 0");
  DB200_REQUIRE(dh == 64 || dh == 128, DB200_E_UNSUPPORTED, "attn: head_dim %d not in {64,128}", dh);
  const int rc = attn_delta(stream, out, dout, delta, B, S, H, dh);
  if (rc != DB200_OK) return rc;
  return attn_axial_bwd_launch(stream, qkv, dout, lse, delta, dqkv, B, S, H, dh, text_len, grid_w, axis, scale);
}

// ---- convolutional attention of DALL-E image tokens: text queries are causal; an image query at grid row r, column c
// sees every text key and the image keys (r', c') with r - kernel < r' <= r and c - kernel < c' <= c.
// S <= text_len + grid_w^2 (a prefill may be shorter).  No dropout.
static int conv_args_ok(const char* fn, int S, int text_len, int grid_w, int kernel) {
  DB200_REQUIRE(kernel >= 1, DB200_E_INVALID, "%s: kernel %d < 1", fn, kernel);
  DB200_REQUIRE(grid_w >= 1 && text_len >= 0, DB200_E_INVALID, "%s: grid_w %d < 1 or text_len %d < 0", fn, grid_w,
                text_len);
  DB200_REQUIRE((long long)S <= (long long)text_len + (long long)grid_w * grid_w, DB200_E_INVALID,
                "%s: S %d exceeds text_len %d + grid_w^2 (%d^2)", fn, S, text_len, grid_w);
  return DB200_OK;
}

extern "C" int db200_attn_conv_fwd(db200_stream_t stream_, const void* qkv, void* out, float* lse, int B, int S, int H,
                                   int dh, int text_len, int grid_w, int kernel, float scale) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && S > 0 && H > 0, DB200_E_INVALID, "attn_conv_fwd: B,S,H must be positive");
  const int arc = conv_args_ok("attn_conv_fwd", S, text_len, grid_w, kernel);
  if (arc != DB200_OK) return arc;
  DB200_REQUIRE(qkv && out && lse && aligned16(qkv) && aligned16(out), DB200_E_ALIGN,
                "attn_conv_fwd: NULL or unaligned pointer");
  DB200_REQUIRE(scale > 0.f, DB200_E_INVALID, "attn_conv_fwd: scale must be > 0");
  DB200_REQUIRE(dh == 64 || dh == 128, DB200_E_UNSUPPORTED, "attn: head_dim %d not in {64,128}", dh);
  return attn_conv_fwd_launch(stream, qkv, out, lse, B, S, H, dh, text_len, grid_w, kernel, scale);
}

extern "C" int db200_attn_conv_bwd(db200_stream_t stream_, const void* qkv, const void* out, const void* dout,
                                   const float* lse, float* dq_accum, float* delta, void* dqkv, int B, int S, int H,
                                   int dh, int text_len, int grid_w, int kernel, float scale) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  (void)dq_accum;
  DB200_REQUIRE(B > 0 && S > 0 && H > 0, DB200_E_INVALID, "attn_conv_bwd: B,S,H must be positive");
  const int arc = conv_args_ok("attn_conv_bwd", S, text_len, grid_w, kernel);
  if (arc != DB200_OK) return arc;
  DB200_REQUIRE(qkv && out && dout && lse && delta && dqkv && aligned16(qkv) && aligned16(out) && aligned16(dout) &&
                    aligned16(dqkv),
                DB200_E_ALIGN, "attn_conv_bwd: NULL or unaligned pointer");
  DB200_REQUIRE(scale > 0.f, DB200_E_INVALID, "attn_conv_bwd: scale must be > 0");
  DB200_REQUIRE(dh == 64 || dh == 128, DB200_E_UNSUPPORTED, "attn: head_dim %d not in {64,128}", dh);
  const int rc = attn_delta(stream, out, dout, delta, B, S, H, dh);
  if (rc != DB200_OK) return rc;
  return attn_conv_bwd_launch(stream, qkv, dout, lse, delta, dqkv, B, S, H, dh, text_len, grid_w, kernel, scale);
}

// ---- block-sparse attention: the 16-bit tile masks of a [>= ceil(S / 64)] x pitch table (attn_fa.cu, SPARSE) under
// the causal mask.  No dropout.
extern "C" int db200_attn_block_sparse_fwd(db200_stream_t stream_, const void* qkv, void* out, float* lse, int B, int S,
                                           int H, int dh, const uint16_t* tile_mask, int mask_pitch, float scale) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && S > 0 && H > 0, DB200_E_INVALID, "attn_block_sparse_fwd: B,S,H must be positive");
  DB200_REQUIRE(tile_mask && mask_pitch >= (S + 63) / 64, DB200_E_INVALID,
                "attn_block_sparse_fwd: NULL tile mask or pitch %d < ceil(S / 64) for S %d", mask_pitch, S);
  DB200_REQUIRE(qkv && out && lse && aligned16(qkv) && aligned16(out), DB200_E_ALIGN,
                "attn_block_sparse_fwd: NULL or unaligned pointer");
  DB200_REQUIRE(scale > 0.f, DB200_E_INVALID, "attn_block_sparse_fwd: scale must be > 0");
  DB200_REQUIRE(dh == 64 || dh == 128, DB200_E_UNSUPPORTED, "attn: head_dim %d not in {64,128}", dh);
  return attn_block_sparse_fwd_launch(stream, qkv, out, lse, B, S, H, dh, tile_mask, mask_pitch, scale);
}

extern "C" int db200_attn_block_sparse_bwd(db200_stream_t stream_, const void* qkv, const void* out, const void* dout,
                                           const float* lse, float* dq_accum, float* delta, void* dqkv, int B, int S,
                                           int H, int dh, const uint16_t* tile_mask, int mask_pitch, float scale) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  (void)dq_accum;
  DB200_REQUIRE(B > 0 && S > 0 && H > 0, DB200_E_INVALID, "attn_block_sparse_bwd: B,S,H must be positive");
  DB200_REQUIRE(tile_mask && mask_pitch >= (S + 63) / 64, DB200_E_INVALID,
                "attn_block_sparse_bwd: NULL tile mask or pitch %d < ceil(S / 64) for S %d", mask_pitch, S);
  DB200_REQUIRE(qkv && out && dout && lse && delta && dqkv && aligned16(qkv) && aligned16(out) && aligned16(dout) &&
                    aligned16(dqkv),
                DB200_E_ALIGN, "attn_block_sparse_bwd: NULL or unaligned pointer");
  DB200_REQUIRE(scale > 0.f, DB200_E_INVALID, "attn_block_sparse_bwd: scale must be > 0");
  DB200_REQUIRE(dh == 64 || dh == 128, DB200_E_UNSUPPORTED, "attn: head_dim %d not in {64,128}", dh);
  const int rc = attn_delta(stream, out, dout, delta, B, S, H, dh);
  if (rc != DB200_OK) return rc;
  return attn_block_sparse_bwd_launch(stream, qkv, dout, lse, delta, dqkv, B, S, H, dh, tile_mask, mask_pitch, scale);
}
