// K14 — the pieces of a taming-transformers VQGAN's forward that the convolutions (K11) and the GEMM do not cover:
// GroupNorm on NHWC bf16 activations (fp32 statistics, optional fused swish), the AttnBlock's non-causal single-head
// attention over one image's positions, and the exact gather of codebook rows for decoding.  Forward only: the
// tokenizer is used frozen.  No float atomics anywhere, so every result is bit-reproducible and an image's result does
// not depend on the batch it is computed in (every launch geometry below depends on H*W and C, never on N).
#include "common.cuh"

namespace db200 {

constexpr int GN_THREADS = 256;
constexpr int GN_ITERS = 16;  // pixel rows each thread reads per chunk

// pixel rows read at once by one CTA: C / 8 threads cover one row of C channels with 16-byte loads
static inline int gn_rows_per_iter(int C) { return GN_THREADS / (C / 8); }
static inline int gn_chunks(int HW, int C) {
  const int ppc = gn_rows_per_iter(C) * GN_ITERS;
  return (HW + ppc - 1) / ppc;
}

// (count, mean, M2) states combined with Chan et al.'s pairwise update
struct Welford {
  float n, m, M2;
};
__device__ __forceinline__ void chan_add(Welford& a, const Welford& b) {
  if (b.n == 0.f) return;
  const float n = a.n + b.n, d = b.m - a.m, f = b.n / n;
  a.m = fmaf(d, f, a.m);
  a.M2 = a.M2 + b.M2 + d * d * a.n * f;
  a.n = n;
}

// One CTA = (image n, chunk of pixel rows).  Each thread keeps a Welford state per channel for its 8 channels over the
// rows it reads (same count for all 8); then, for each group, one thread combines the group's per-(thread, channel)
// states in a fixed order and stores the chunk's (count, mean, M2) into the workspace.
__global__ void __launch_bounds__(GN_THREADS)
groupnorm_partial_kernel(const bf16* __restrict__ x, float* __restrict__ part, int HW, int C, int G, int chunks) {
  extern __shared__ float gn_smem[];
  const int tpr = C / 8, rpi = GN_THREADS / tpr;
  float* s_m = gn_smem;                    // [rpi * tpr][8]
  float* s_M2 = s_m + GN_THREADS * 8;      // [rpi * tpr][8]
  float* s_n = s_M2 + GN_THREADS * 8;      // [rpi * tpr]
  const int n = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
  const int row = tid / tpr, col = tid % tpr;
  const int p0 = chunk * rpi * GN_ITERS, p1 = min(HW, p0 + rpi * GN_ITERS);
  float m[8], M2[8], cnt = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) m[j] = M2[j] = 0.f;
  if (row < rpi) {
    const bf16* base = x + (long long)n * HW * C + col * 8;
    for (int p = p0 + row; p < p1; p += rpi) {
      const uint4 v = *reinterpret_cast<const uint4*>(base + (long long)p * C);
      const bf16* e = reinterpret_cast<const bf16*>(&v);
      cnt += 1.f;
      const float inv = 1.f / cnt;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xv = __bfloat162float(e[j]);
        const float d = xv - m[j];
        m[j] = fmaf(d, inv, m[j]);
        M2[j] = fmaf(d, xv - m[j], M2[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s_m[tid * 8 + j] = m[j];
      s_M2[tid * 8 + j] = M2[j];
    }
    s_n[tid] = cnt;
  }
  __syncthreads();
  const int cg = C / G;
  for (int g = tid; g < G; g += GN_THREADS) {
    Welford acc{0.f, 0.f, 0.f};
    for (int r = 0; r < rpi; ++r)
      for (int c = g * cg; c < (g + 1) * cg; ++c) {
        const int t = r * tpr + c / 8;
        chan_add(acc, Welford{s_n[t], s_m[t * 8 + (c & 7)], s_M2[t * 8 + (c & 7)]});
      }
    float* o = part + (((long long)n * chunks + chunk) * G + g) * 3;
    o[0] = acc.n; o[1] = acc.m; o[2] = acc.M2;
  }
}

// one thread per (image, group): the chunks' states combined in chunk order, biased variance
__global__ void groupnorm_finish_kernel(const float* __restrict__ part, float* __restrict__ mean,
                                        float* __restrict__ rstd, int N, int G, int chunks, float eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * G) return;
  const int n = i / G, g = i % G;
  Welford acc{0.f, 0.f, 0.f};
  for (int c = 0; c < chunks; ++c) {
    const float* p = part + (((long long)n * chunks + c) * G + g) * 3;
    chan_add(acc, Welford{p[0], p[1], p[2]});
  }
  mean[i] = acc.m;
  rstd[i] = 1.f / sqrtf(acc.M2 / acc.n + eps);
}

// y = (x - mean) * rstd * gamma + beta [then swish(v) = v * sigmoid(v)], 8 channels per thread and step
template <bool SWISH>
__global__ void __launch_bounds__(256)
groupnorm_apply_kernel(const bf16* __restrict__ x, const float* __restrict__ mean, const float* __restrict__ rstd,
                       const float* __restrict__ gamma, const float* __restrict__ beta, bf16* __restrict__ y,
                       long long n_vec, int HW, int C, int G) {
  const int cg = C / G, vpr = C / 8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    const long long pix = i / vpr;
    const int c0 = (int)(i % vpr) * 8;
    const int n = (int)(pix / HW);
    const uint4 v = *reinterpret_cast<const uint4*>(x + i * 8);
    const bf16* e = reinterpret_cast<const bf16*>(&v);
    uint4 out;
    bf16* o = reinterpret_cast<bf16*>(&out);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c0 + j, s = n * G + c / cg;
      float t = (__bfloat162float(e[j]) - mean[s]) * rstd[s] * gamma[c] + beta[c];
      if (SWISH) t = t / (1.f + __expf(-t));
      o[j] = __float2bfloat16(t);
    }
    *reinterpret_cast<uint4*>(y + i * 8) = out;
  }
}

// ---- non-causal single-head attention: o_i = sum_j softmax_j(scale q_i . k_j) v_j over one image's S positions ----
constexpr int AT_THREADS = 256;
constexpr int AT_BQ = 32;    // queries per CTA
constexpr int AT_KC = 32;    // channels of q / k staged per step of the score product
constexpr int AT_VS = 32;    // positions of v staged per step of the weighted sum
constexpr int AT_VC = 64;    // output columns per pass of the weighted sum
constexpr int AT_SMAX = 256;
constexpr int AT_PLD = AT_SMAX + 4;

static inline size_t attn_smem_bytes() {
  const size_t p = (size_t)AT_BQ * AT_PLD;
  const size_t qk = (size_t)AT_KC * AT_BQ + (size_t)AT_KC * (AT_SMAX + 1);
  const size_t v = (size_t)AT_VS * AT_VC;
  return (p + (qk > v ? qk : v)) * sizeof(float);
}

// One CTA = (image b, 32 queries).  The whole score row of each query (S <= 256) stays in shared memory in fp32:
//   1. scores: warp w owns queries 4w..4w+3, lane l keys l, l + 32, ...; q and k are staged 32 channels at a time
//      (k transposed, so a warp reads 32 consecutive keys);
//   2. softmax per row with the row maximum subtracted, sums reduced by a fixed shuffle tree;
//   3. o = P v in passes of 64 output columns (C up to 512 would not fit in registers at once): thread (ty, tx) owns
//      queries 2ty, 2ty + 1 and columns 4tx..4tx+3 of the pass.
__global__ void __launch_bounds__(AT_THREADS)
attn_noncausal_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ out, int S, int C, float scale) {
  extern __shared__ float at_smem[];
  float* P = at_smem;                       // [AT_BQ][AT_PLD]
  float* Qs = P + AT_BQ * AT_PLD;           // [AT_KC][AT_BQ]
  float* Ks = Qs + AT_KC * AT_BQ;           // [AT_KC][AT_SMAX + 1]
  float* Vs = Qs;                           // [AT_VS][AT_VC] (phase 3 reuses the q / k staging area)
  const int b = blockIdx.y, q0 = blockIdx.x * AT_BQ, tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const long long ld = 3ll * C;
  const bf16* base = qkv + (long long)b * S * ld;
  const int nk = S / 32;

  float acc[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  for (int c0 = 0; c0 < C; c0 += AT_KC) {
    {  // q: 32 rows x 32 channels, 4 channels per thread
      const int r = tid >> 3, c = (tid & 7) * 4;
      const bf16* src = base + (long long)(q0 + r) * ld + c0 + c;
#pragma unroll
      for (int j = 0; j < 4; ++j) Qs[(c + j) * AT_BQ + r] = __bfloat162float(src[j]);
    }
    for (int r = tid >> 2; r < S; r += AT_THREADS / 4) {  // k: S rows x 32 channels, 8 channels per thread
      const int c = (tid & 3) * 8;
      const uint4 v = *reinterpret_cast<const uint4*>(base + (long long)r * ld + C + c0 + c);
      const bf16* e = reinterpret_cast<const bf16*>(&v);
#pragma unroll
      for (int j = 0; j < 8; ++j) Ks[(c + j) * (AT_SMAX + 1) + r] = __bfloat162float(e[j]);
    }
    __syncthreads();
#pragma unroll 4
    for (int c = 0; c < AT_KC; ++c) {
      const float4 q = *reinterpret_cast<const float4*>(&Qs[c * AT_BQ + warp * 4]);
      const float qv[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (j < nk) {
          const float kv = Ks[c * (AT_SMAX + 1) + lane + 32 * j];
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[i][j] = fmaf(qv[i], kv, acc[i][j]);
        }
      }
    }
    __syncthreads();
  }
  // softmax of each of this warp's 4 rows
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < nk) mx = fmaxf(mx, acc[i][j] * scale);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < nk) {
        acc[i][j] = expf(acc[i][j] * scale - mx);
        sum += acc[i][j];
      }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.f / sum;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < nk) P[(warp * 4 + i) * AT_PLD + lane + 32 * j] = acc[i][j] * inv;
  }
  __syncthreads();
  const int tx = tid & 15, ty = tid >> 4;
  for (int n0 = 0; n0 < C; n0 += AT_VC) {
    float o[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
    for (int s0 = 0; s0 < S; s0 += AT_VS) {
      {  // v: 32 rows x 64 columns, 8 columns per thread
        const int r = tid >> 3, c = (tid & 7) * 8;
        const uint4 v = *reinterpret_cast<const uint4*>(base + (long long)(s0 + r) * ld + 2 * C + n0 + c);
        const bf16* e = reinterpret_cast<const bf16*>(&v);
#pragma unroll
        for (int j = 0; j < 8; ++j) Vs[r * AT_VC + c + j] = __bfloat162float(e[j]);
      }
      __syncthreads();
#pragma unroll 8
      for (int s = 0; s < AT_VS; ++s) {
        const float4 v = *reinterpret_cast<const float4*>(&Vs[s * AT_VC + tx * 4]);
        const float p0 = P[(2 * ty) * AT_PLD + s0 + s], p1 = P[(2 * ty + 1) * AT_PLD + s0 + s];
        o[0][0] = fmaf(p0, v.x, o[0][0]); o[0][1] = fmaf(p0, v.y, o[0][1]);
        o[0][2] = fmaf(p0, v.z, o[0][2]); o[0][3] = fmaf(p0, v.w, o[0][3]);
        o[1][0] = fmaf(p1, v.x, o[1][0]); o[1][1] = fmaf(p1, v.y, o[1][1]);
        o[1][2] = fmaf(p1, v.z, o[1][2]); o[1][3] = fmaf(p1, v.w, o[1][3]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      bf16* dst = out + ((long long)b * S + q0 + 2 * ty + i) * C + n0 + tx * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) dst[j] = __float2bfloat16(o[i][j]);
    }
  }
}

// hi = bf16(table[idx - offset]), lo = bf16(row - hi); rows whose id is outside [offset, offset + K) get zeros
__global__ void gather_rows_split_kernel(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                         bf16* __restrict__ hi, bf16* __restrict__ lo, long long n, int D, int K,
                                         int offset) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / D;
    const int id = idx[r] - offset;
    const float v = (id >= 0 && id < K) ? table[(long long)id * D + (i % D)] : 0.f;
    const bf16 h = __float2bfloat16(v);
    hi[i] = h;
    if (lo) lo[i] = __float2bfloat16(v - __bfloat162float(h));
  }
}

// dst = clamp(float(src), lo, hi): the decoder's bf16 output as the caller's f32 image
__global__ void clamp_bf16_to_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst, long long n, float lo,
                                         float hi) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = fminf(fmaxf(__bfloat162float(src[i]), lo), hi);
}

static int grid_for(long long work, int threads) {
  long long g = (work + threads - 1) / threads;
  const long long cap = (long long)sm_count() * 16;
  if (g > cap) g = cap;
  return (int)(g < 1 ? 1 : g);
}

static int gn_check(const char* who, int N, int HW, int C, int G) {
  DB200_REQUIRE(N > 0 && HW > 0 && C > 0 && G > 0, DB200_E_INVALID, "%s: non-positive dimension", who);
  DB200_REQUIRE(C % 8 == 0 && C % G == 0 && C <= 8 * GN_THREADS, DB200_E_UNSUPPORTED,
                "%s: C = %d must be a multiple of 8 and of G = %d, and at most %d", who, C, G, 8 * GN_THREADS);
  return DB200_OK;
}

}  // namespace db200

using namespace db200;

extern "C" int64_t db200_groupnorm_stats_workspace_bytes(int N, int HW, int C, int G) {
  if (gn_check("groupnorm_stats", N, HW, C, G) != DB200_OK) return 0;
  return (int64_t)N * gn_chunks(HW, C) * G * 3 * sizeof(float);
}

extern "C" int db200_groupnorm_stats(db200_stream_t stream_, const void* x, float* mean, float* rstd, int N, int HW,
                                     int C, int G, float eps, void* workspace, int64_t workspace_bytes) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = gn_check("groupnorm_stats", N, HW, C, G);
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(x && mean && rstd, DB200_E_INVALID, "groupnorm_stats: NULL pointer");
  DB200_REQUIRE(aligned16(x), DB200_E_ALIGN, "groupnorm_stats: x must be 16-byte aligned");
  DB200_REQUIRE(eps >= 0.f, DB200_E_INVALID, "groupnorm_stats: eps < 0");
  const int chunks = gn_chunks(HW, C);
  DB200_REQUIRE(workspace_ok(workspace, workspace_bytes, db200_groupnorm_stats_workspace_bytes(N, HW, C, G)),
                DB200_E_INVALID, "groupnorm_stats: workspace too small or unaligned");
  DB200_REQUIRE(N <= 65535, DB200_E_UNSUPPORTED, "groupnorm_stats: N = %d > 65535", N);
  float* part = reinterpret_cast<float*>(workspace);
  const size_t smem = (size_t)GN_THREADS * 17 * sizeof(float);
  groupnorm_partial_kernel<<<dim3(chunks, N), GN_THREADS, smem, stream>>>(reinterpret_cast<const bf16*>(x), part, HW,
                                                                          C, G, chunks);
  rc = check_launch("groupnorm_partial_kernel");
  if (rc != DB200_OK) return rc;
  groupnorm_finish_kernel<<<(N * G + 127) / 128, 128, 0, stream>>>(part, mean, rstd, N, G, chunks, eps);
  return check_launch("groupnorm_finish_kernel");
}

extern "C" int db200_groupnorm_apply(db200_stream_t stream_, const void* x, const float* mean, const float* rstd,
                                     const float* gamma, const float* beta, void* y, int N, int HW, int C, int G,
                                     int swish) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = gn_check("groupnorm_apply", N, HW, C, G);
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(x && mean && rstd && gamma && beta && y, DB200_E_INVALID, "groupnorm_apply: NULL pointer");
  DB200_REQUIRE(aligned16(x) && aligned16(y), DB200_E_ALIGN, "groupnorm_apply: x and y must be 16-byte aligned");
  const long long n_vec = (long long)N * HW * (C / 8);
  const int grid = grid_for(n_vec, 256);
  const bf16* xb = reinterpret_cast<const bf16*>(x);
  bf16* yb = reinterpret_cast<bf16*>(y);
  if (swish) groupnorm_apply_kernel<true><<<grid, 256, 0, stream>>>(xb, mean, rstd, gamma, beta, yb, n_vec, HW, C, G);
  else       groupnorm_apply_kernel<false><<<grid, 256, 0, stream>>>(xb, mean, rstd, gamma, beta, yb, n_vec, HW, C, G);
  return check_launch("groupnorm_apply_kernel");
}

extern "C" int db200_attn_noncausal_fwd(db200_stream_t stream_, const void* qkv, void* out, int B, int S, int C,
                                        float scale) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(qkv && out && B > 0 && S > 0 && C > 0, DB200_E_INVALID, "attn_noncausal_fwd: bad arguments");
  DB200_REQUIRE(S % 64 == 0 && S <= AT_SMAX && C % 64 == 0 && C <= 512 && B <= 65535, DB200_E_UNSUPPORTED,
                "attn_noncausal_fwd: S = %d must be a multiple of 64 up to %d and C = %d a multiple of 64 up to 512",
                S, AT_SMAX, C);
  DB200_REQUIRE(aligned16(qkv) && aligned16(out), DB200_E_ALIGN, "attn_noncausal_fwd: pointers must be 16-byte aligned");
  const size_t smem = attn_smem_bytes();
  DB200_CUDA(cudaFuncSetAttribute(attn_noncausal_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  attn_noncausal_kernel<<<dim3(S / AT_BQ, B), AT_THREADS, smem, stream>>>(reinterpret_cast<const bf16*>(qkv),
                                                                          reinterpret_cast<bf16*>(out), S, C, scale);
  return check_launch("attn_noncausal_kernel");
}

extern "C" int db200_gather_rows_split(db200_stream_t stream_, const int32_t* idx, const float* table, void* hi,
                                       void* lo_or_null, int rows, int D, int K, int offset) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(idx && table && hi && rows > 0 && D > 0 && K > 0, DB200_E_INVALID, "gather_rows_split: bad arguments");
  const long long n = (long long)rows * D;
  gather_rows_split_kernel<<<grid_for(n, 256), 256, 0, stream>>>(idx, table, reinterpret_cast<bf16*>(hi),
                                                                  reinterpret_cast<bf16*>(lo_or_null), n, D, K, offset);
  return check_launch("gather_rows_split_kernel");
}

extern "C" int db200_clamp_bf16_to_f32(db200_stream_t stream_, const void* src, float* dst, int64_t n, float lo,
                                       float hi) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(src && dst && n > 0 && lo <= hi, DB200_E_INVALID, "clamp_bf16_to_f32: bad arguments");
  clamp_bf16_to_f32_kernel<<<grid_for(n, 256), 256, 0, stream>>>(reinterpret_cast<const bf16*>(src), dst, n, lo, hi);
  return check_launch("clamp_bf16_to_f32_kernel");
}
