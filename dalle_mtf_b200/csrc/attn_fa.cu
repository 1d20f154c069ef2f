// K4 — causal flash attention on wgmma (sm_90a): forward, and the backward as two kernels (dQ per query block, dK / dV
// per key block), so that no gradient needs atomics.
//
// One CTA = one warpgroup = 64 rows of one (batch, head).  Tiles of 64 rows x dh are brought into shared memory with
// cp.async in the 128B-swizzled layout of the wgmma descriptors ([dh / 64 atoms][64 rows][64 bf16]); the same K / V /
// Q / dO tile serves as a K-major operand (rows = the contracted dimension's partner) and, read through an MN-major
// descriptor, as the B operand of the products that contract over its rows.  Logits, softmax and gradients stay in the
// fp32 accumulator fragments; P and dS are packed to bf16 in registers and fed to the next wgmma as its A operand.
//
// Layout: qkv bf16 [B][S][3][H][dh], out / dout bf16 [B][S][H][dh], lse / delta f32 [B][H][S], dqkv like qkv.
//
// LOCAL (sliding-window attention, mtf local_attention_1d with fully_autoregressive=True, src/dalle_mtf/models.py:
// 257-273): query i sees key j iff i - radius < j <= i.  The loops visit only the key (query) blocks that intersect that
// band and the masks add the lower edge; the global (causal) instantiations compile without either.
#include "gemm_common.cuh"  // cp.async helpers
#include "philox.cuh"
#include "wgmma.cuh"

namespace db200 {
namespace {

constexpr int FA_ROWS = 64;
constexpr float kLn2 = 0.6931471805599453f;

// 64 rows x DH bf16 (row r at src + r * ld, rows >= n_rows zero-filled) -> swizzled smem tile; the caller commits
template <int DH>
__device__ __forceinline__ void fa_load_tile(uint32_t dst, const bf16* src, long long ld, int n_rows) {
  constexpr int CPR = DH / 8;  // 16-byte chunks per row
#pragma unroll
  for (int i = 0; i < FA_ROWS * CPR / 128; ++i) {
    const int idx = threadIdx.x + 128 * i;
    const int r = idx / CPR, c = idx % CPR;
    const bool ok = r < n_rows;
    const uint32_t off = (c >> 3) * (FA_ROWS * 128) + r * 128 + ((((c & 7) ^ (r & 7)) & 7) << 4);
    cp_async16_zfill(dst + off, ok ? src + (long long)r * ld + c * 8 : src, ok);
  }
}
// all outstanding tile loads have landed and are visible to the wgmma (async) proxy of every thread
__device__ __forceinline__ void fa_tiles_ready() {
  cp_async_commit();
  cp_async_wait<0>();
  fence_proxy_async_smem();
  __syncthreads();
}

// K-major descriptor of k-step ks (16 columns) of a [64 rows][DH] tile: 64-column atoms 8 KiB apart
__device__ __forceinline__ uint64_t fa_kdesc(uint32_t tile, int ks) {
  return smem_desc_sw128(tile + (ks >> 2) * (FA_ROWS * 128) + (ks & 3) * 32, 0, 1024);
}
// MN-major descriptor of k-step ks (16 rows) of the same tile used as a B operand with N = DH
__device__ __forceinline__ uint64_t fa_ndesc(uint32_t tile, int ks) {
  return smem_desc_sw128(tile + ks * 2048, FA_ROWS * 128, 1024);
}

// S[64 x 64] = A_tile[64 x DH] * B_tile[64 x DH]^T (both K-major)
template <int DH>
__device__ __forceinline__ void fa_qk(float* s, uint32_t a_tile, uint32_t b_tile) {
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < DH / 16; ++ks) wgmma_m64n64<0, 0>(s, fa_kdesc(a_tile, ks), fa_kdesc(b_tile, ks), ks > 0);
  wgmma_commit();
  wgmma_wait<0>();
}
// acc[64 x DH] += P[64 x 64] (registers, fp32 fragment packed to bf16 here) * tile[64 x DH]
// DROP: fragment element x is multiplied by (bit x of kb) ? sc : 0 on the way (dropout of P)
template <int DH, bool DROP = false>
__device__ __forceinline__ void fa_pv(float* acc, const float* p, uint32_t tile, uint32_t kb = 0u, float sc = 1.f) {
  uint32_t a[4][4];
  auto pk = [&](int x) { return DROP ? (((kb >> x) & 1u) ? p[x] * sc : 0.f) : p[x]; };
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = pack_bf16x2(pk(8 * ks + 0), pk(8 * ks + 1));
    a[ks][1] = pack_bf16x2(pk(8 * ks + 2), pk(8 * ks + 3));
    a[ks][2] = pack_bf16x2(pk(8 * ks + 4), pk(8 * ks + 5));
    a[ks][3] = pack_bf16x2(pk(8 * ks + 6), pk(8 * ks + 7));
  }
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    if constexpr (DH == 64) wgmma_rs_m64n64<1>(acc, a[ks], fa_ndesc(tile, ks), 1u);
    else wgmma_rs_m64n128<1>(acc, a[ks], fa_ndesc(tile, ks), 1u);
  }
  wgmma_commit();
  wgmma_wait<0>();
}

// fragment coordinates: element (i, h, e) of an m64 x N accumulator sits at row fr + 8 h, column 8 i + fc + e
struct Frag {
  int fr, fc;
  __device__ __forceinline__ Frag() {
    const int t = threadIdx.x & 127, lane = t & 31;
    fr = 16 * (t >> 5) + (lane >> 2);
    fc = 2 * (lane & 3);
  }
};
// Keep bits of this thread's 32 fragment elements of a 64 x 64 attention-weight tile (bit x = element x) whose first
// row / column are r0 / c0.  QROWS: rows are queries and columns keys (forward, dQ); else rows are keys and columns
// queries (dK / dV).  The two columns fc, fc + 1 of a row share one 2 x 2 block, so each Philox call serves two elements.
template <bool QROWS>
__device__ __forceinline__ uint32_t fa_keep_bits(const db200_dropout& dr, int b, int h, int H, int S2, int r0, int c0,
                                                 const Frag& f) {
  uint32_t kb = 0u;
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = r0 + f.fr + 8 * hh, col = c0 + 8 * i + f.fc;  // col is even
      const uint4 r = dropout_block(dr, QROWS ? dropout_attn_block(dr, b, h, H, S2, row, col)
                                              : dropout_attn_block(dr, b, h, H, S2, col, row));
      // word of (query i, key j) = 2 (i & 1) + (j & 1)
      const uint32_t w0 = QROWS ? ((row & 1) ? r.z : r.x) : ((row & 1) ? r.y : r.x);
      const uint32_t w1 = QROWS ? ((row & 1) ? r.w : r.y) : ((row & 1) ? r.w : r.z);
      const int x = 4 * i + 2 * hh;
      kb |= (uint32_t)(w0 >= dr.threshold) << x;
      kb |= (uint32_t)(w1 >= dr.threshold) << (x + 1);
    }
  return kb;
}
__device__ __forceinline__ float fa_keep_mul(uint32_t kb, int x, float sc) { return ((kb >> x) & 1u) ? sc : 0.f; }

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// store an m64 x DH fp32 fragment (times `mul`) as bf16 rows r < n_rows of dst (row stride ld)
template <int DH>
__device__ __forceinline__ void fa_store_rows(bf16* dst, long long ld, const float* acc, const float (&mul)[2],
                                              int n_rows, const Frag& f) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = f.fr + 8 * h;
    if (r >= n_rows) continue;
    bf16* d = dst + (long long)r * ld + f.fc;
#pragma unroll
    for (int i = 0; i < DH / 8; ++i)
      *reinterpret_cast<uint32_t*>(d + 8 * i) = pack_bf16x2(acc[4 * i + 2 * h] * mul[h], acc[4 * i + 2 * h + 1] * mul[h]);
  }
}

template <int DH>
constexpr size_t fa_smem(int tiles) { return 1024 + size_t(tiles) * FA_ROWS * DH * 2 + 2 * FA_ROWS * 4; }

}  // namespace

// ------------------------------------------------------------------------------------------------------------------
// forward: grid (query blocks, B * H); online softmax in the exp2 domain
// ------------------------------------------------------------------------------------------------------------------
template <int DH, bool DROP, bool LOCAL>
__global__ void __launch_bounds__(128, 1)
attn_fwd_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ out, float* __restrict__ lse, int S, int H,
                float scale, const db200_dropout dr, int radius) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t TILE = FA_ROWS * DH * 2;
  const uint32_t sQ = base, sK = base + TILE, sV = base + 2 * TILE;
  const int qb = blockIdx.x, b = blockIdx.y / H, h = blockIdx.y % H;
  const int q0 = qb * FA_ROWS;
  const long long ldq = 3LL * H * DH;
  const bf16* Q = qkv + (long long)b * S * ldq + (long long)h * DH;
  const Frag f;
  const float sl2 = scale * kLog2e;

  fa_load_tile<DH>(sQ, Q + q0 * ldq, ldq, S - q0);
  float o[DH / 2], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
  const int j0 = LOCAL ? max(0, q0 - radius + 1) / FA_ROWS : 0;
  for (int j = j0; j <= qb; ++j) {
    const int k0 = j * FA_ROWS;
    __syncthreads();  // the previous block's K / V tiles are no longer read
    fa_load_tile<DH>(sK, Q + k0 * ldq + (long long)H * DH, ldq, S - k0);
    fa_load_tile<DH>(sV, Q + k0 * ldq + 2LL * H * DH, ldq, S - k0);
    fa_tiles_ready();
    float s[32];
    fa_qk<DH>(s, sQ, sK);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int row = q0 + f.fr + 8 * hh, col = k0 + 8 * i + f.fc + e;
          float& v = s[4 * i + 2 * hh + e];
          v = (col <= row && col < S && (!LOCAL || col > row - radius)) ? v * sl2 : -INFINITY;
          mx[hh] = fmaxf(mx[hh], v);
        }
    float alpha[2], mb[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const float mn = fmaxf(m[hh], quad_max(mx[hh]));
      mb[hh] = mn == -INFINITY ? 0.f : mn;
      alpha[hh] = exp2f(m[hh] - mb[hh]);
      m[hh] = mn;
      l[hh] *= alpha[hh];
    }
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) {
      o[4 * i + 0] *= alpha[0]; o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
    }
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = s[4 * i + 2 * hh + e];
          v = exp2f(v - mb[hh]);
          l[hh] += v;
        }
    // l (hence lse) sums the undropped weights; dropout acts on the normalised weights, i.e. on P before PV
    if constexpr (DROP)
      fa_pv<DH, true>(o, s, sV, fa_keep_bits<true>(dr, b, h, H, (S + 1) >> 1, q0, k0, f), dr.scale);
    else
      fa_pv<DH>(o, s, sV);
  }
  float inv[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float tot = quad_sum(l[hh]);
    inv[hh] = tot > 0.f ? 1.f / tot : 0.f;
    const int row = q0 + f.fr + 8 * hh;
    if ((f.fc == 0) && row < S) lse[((long long)b * H + h) * S + row] = (m[hh] + log2f(tot)) * kLn2;
  }
  fa_store_rows<DH>(out + ((long long)b * S + q0) * H * DH + (long long)h * DH, (long long)H * DH, o, inv, S - q0, f);
}

// ------------------------------------------------------------------------------------------------------------------
// backward, dQ: grid (query blocks, B * H).  P = exp(scale S - lse), dS = P (dO V^T - delta), dQ = scale dS K
// ------------------------------------------------------------------------------------------------------------------
template <int DH, bool DROP, bool LOCAL>
__global__ void __launch_bounds__(128, 1)
attn_bwd_dq_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ dout, const float* __restrict__ lse,
                   const float* __restrict__ delta, bf16* __restrict__ dqkv, int S, int H, float scale,
                   const db200_dropout dr, int radius) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t TILE = FA_ROWS * DH * 2;
  const uint32_t sQ = base, sdO = base + TILE, sK = base + 2 * TILE, sV = base + 3 * TILE;
  const int qb = blockIdx.x, b = blockIdx.y / H, h = blockIdx.y % H;
  const int q0 = qb * FA_ROWS;
  const long long ldq = 3LL * H * DH, ldo = (long long)H * DH;
  const bf16* Q = qkv + (long long)b * S * ldq + (long long)h * DH;
  const Frag f;
  const float sl2 = scale * kLog2e;

  fa_load_tile<DH>(sQ, Q + q0 * ldq, ldq, S - q0);
  fa_load_tile<DH>(sdO, dout + ((long long)b * S + q0) * ldo + (long long)h * DH, ldo, S - q0);
  float lse2[2], dl[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = q0 + f.fr + 8 * hh;
    const long long ix = ((long long)b * H + h) * S + (row < S ? row : S - 1);
    lse2[hh] = lse[ix] * kLog2e;
    dl[hh] = delta[ix];
  }
  float dq[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) dq[i] = 0.f;
  const int j0 = LOCAL ? max(0, q0 - radius + 1) / FA_ROWS : 0;
  for (int j = j0; j <= qb; ++j) {
    const int k0 = j * FA_ROWS;
    __syncthreads();
    fa_load_tile<DH>(sK, Q + k0 * ldq + (long long)H * DH, ldq, S - k0);
    fa_load_tile<DH>(sV, Q + k0 * ldq + 2LL * H * DH, ldq, S - k0);
    fa_tiles_ready();
    float s[32], dp[32];
    fa_qk<DH>(s, sQ, sK);
    fa_qk<DH>(dp, sdO, sV);
    // dropout: dS = P (dP keep scale - delta)
    const uint32_t kb = DROP ? fa_keep_bits<true>(dr, b, h, H, (S + 1) >> 1, q0, k0, f) : 0u;
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int row = q0 + f.fr + 8 * hh, col = k0 + 8 * i + f.fc + e;
          const int x = 4 * i + 2 * hh + e;
          const bool vis = col <= row && col < S && row < S && (!LOCAL || col > row - radius);
          const float p = vis ? exp2f(s[x] * sl2 - lse2[hh]) : 0.f;
          s[x] = p * ((DROP ? dp[x] * fa_keep_mul(kb, x, dr.scale) : dp[x]) - dl[hh]);
        }
    fa_pv<DH>(dq, s, sK);
  }
  const float mul[2] = {scale, scale};
  fa_store_rows<DH>(dqkv + ((long long)b * S + q0) * ldq + (long long)h * DH, ldq, dq, mul, S - q0, f);
}

// ------------------------------------------------------------------------------------------------------------------
// backward, dK / dV: grid (key blocks, B * H), transposed products so that the key index is the accumulator row.
//   P^T = exp(scale K Q^T - lse), dV = P^T dO, dS^T = P^T (V dO^T - delta), dK = scale dS^T Q
// ------------------------------------------------------------------------------------------------------------------
template <int DH, bool DROP, bool LOCAL>
__global__ void __launch_bounds__(128, 1)
attn_bwd_dkv_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ dout, const float* __restrict__ lse,
                    const float* __restrict__ delta, bf16* __restrict__ dqkv, int S, int H, float scale,
                    const db200_dropout dr, int radius) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t TILE = FA_ROWS * DH * 2;
  const uint32_t sK = base, sV = base + TILE, sQ = base + 2 * TILE, sdO = base + 3 * TILE;
  float* s_lse = reinterpret_cast<float*>(smem_raw + (base + 4 * TILE - smem_u32(smem_raw)));
  float* s_dl = s_lse + FA_ROWS;
  const int kb = blockIdx.x, b = blockIdx.y / H, h = blockIdx.y % H;
  const int k0 = kb * FA_ROWS;
  const long long ldq = 3LL * H * DH, ldo = (long long)H * DH;
  const bf16* Q = qkv + (long long)b * S * ldq + (long long)h * DH;
  const Frag f;
  const float sl2 = scale * kLog2e;
  // LOCAL: the last query that sees key k0 + 63 is k0 + 62 + radius
  const int nqb = LOCAL ? min((S + FA_ROWS - 1) / FA_ROWS, (int)(((long long)k0 + 62 + radius) / FA_ROWS) + 1)
                        : (S + FA_ROWS - 1) / FA_ROWS;

  fa_load_tile<DH>(sK, Q + k0 * ldq + (long long)H * DH, ldq, S - k0);
  fa_load_tile<DH>(sV, Q + k0 * ldq + 2LL * H * DH, ldq, S - k0);
  float dk[DH / 2], dv[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) { dk[i] = 0.f; dv[i] = 0.f; }
  for (int i = kb; i < nqb; ++i) {
    const int q0 = i * FA_ROWS;
    __syncthreads();
    fa_load_tile<DH>(sQ, Q + q0 * ldq, ldq, S - q0);
    fa_load_tile<DH>(sdO, dout + ((long long)b * S + q0) * ldo + (long long)h * DH, ldo, S - q0);
    if (threadIdx.x < FA_ROWS) {
      const int q = q0 + threadIdx.x;
      const long long ix = ((long long)b * H + h) * S + (q < S ? q : S - 1);
      s_lse[threadIdx.x] = lse[ix] * kLog2e;
      s_dl[threadIdx.x] = delta[ix];
    }
    fa_tiles_ready();
    float st[32], dpt[32];
    fa_qk<DH>(st, sK, sQ);
#pragma unroll
    for (int ii = 0; ii < 8; ++ii)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = k0 + f.fr + 8 * hh, cq = 8 * ii + f.fc + e, q = q0 + cq;
          const int x = 4 * ii + 2 * hh + e;
          const bool vis = key <= q && q < S && key < S && (!LOCAL || key > q - radius);
          st[x] = vis ? exp2f(st[x] * sl2 - s_lse[cq]) : 0.f;
        }
    // dropout: dV += (P keep scale)^T dO,  dS = P (dP keep scale - delta)
    const uint32_t kb = DROP ? fa_keep_bits<false>(dr, b, h, H, (S + 1) >> 1, k0, q0, f) : 0u;
    if constexpr (DROP) fa_pv<DH, true>(dv, st, sdO, kb, dr.scale);
    else fa_pv<DH>(dv, st, sdO);
    fa_qk<DH>(dpt, sV, sdO);
#pragma unroll
    for (int ii = 0; ii < 8; ++ii)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * ii + 2 * hh + e;
          st[x] = st[x] * ((DROP ? dpt[x] * fa_keep_mul(kb, x, dr.scale) : dpt[x]) - s_dl[8 * ii + f.fc + e]);
        }
    fa_pv<DH>(dk, st, sQ);
  }
  const float one[2] = {1.f, 1.f}, mul[2] = {scale, scale};
  bf16* dst = dqkv + ((long long)b * S + k0) * ldq + (long long)h * DH;
  fa_store_rows<DH>(dst + (long long)H * DH, ldq, dk, mul, S - k0, f);
  fa_store_rows<DH>(dst + 2LL * H * DH, ldq, dv, one, S - k0, f);
}

template <int DH, bool DROP, bool LOCAL = false>
static int fa_fwd(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, float scale,
                  const db200_dropout& dr, int radius = 0) {
  constexpr size_t smem = fa_smem<DH>(3);
  static const cudaError_t attr_rc = cudaFuncSetAttribute(attn_fwd_kernel<DH, DROP, LOCAL>,
                                                          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  DB200_CUDA(attr_rc);
  const dim3 grid((S + FA_ROWS - 1) / FA_ROWS, B * H);
  attn_fwd_kernel<DH, DROP, LOCAL><<<grid, 128, smem, stream>>>((const bf16*)qkv, (bf16*)out, lse, S, H, scale, dr,
                                                                radius);
  return check_launch("attn_fwd_kernel");
}

template <int DH, bool DROP, bool LOCAL = false>
static int fa_bwd(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                  void* dqkv, int B, int S, int H, float scale, const db200_dropout& dr, int radius = 0) {
  constexpr size_t smem = fa_smem<DH>(4);
  static const cudaError_t rc1 = cudaFuncSetAttribute(attn_bwd_dq_kernel<DH, DROP, LOCAL>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  static const cudaError_t rc2 = cudaFuncSetAttribute(attn_bwd_dkv_kernel<DH, DROP, LOCAL>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  DB200_CUDA(rc1);
  DB200_CUDA(rc2);
  const dim3 grid((S + FA_ROWS - 1) / FA_ROWS, B * H);
  attn_bwd_dq_kernel<DH, DROP, LOCAL><<<grid, 128, smem, stream>>>((const bf16*)qkv, (const bf16*)dout, lse, delta,
                                                                   (bf16*)dqkv, S, H, scale, dr, radius);
  int rc = check_launch("attn_bwd_dq_kernel");
  if (rc != DB200_OK) return rc;
  attn_bwd_dkv_kernel<DH, DROP, LOCAL><<<grid, 128, smem, stream>>>((const bf16*)qkv, (const bf16*)dout, lse, delta,
                                                                    (bf16*)dqkv, S, H, scale, dr, radius);
  return check_launch("attn_bwd_dkv_kernel");
}

// drop == NULL (or threshold 0): the kernels without dropout
int attn_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, int dh,
                    float scale, const db200_dropout* drop) {
  const db200_dropout none{};
  if (dropout_active(drop))
    return dh == 128 ? fa_fwd<128, true>(stream, qkv, out, lse, B, S, H, scale, *drop)
                     : fa_fwd<64, true>(stream, qkv, out, lse, B, S, H, scale, *drop);
  return dh == 128 ? fa_fwd<128, false>(stream, qkv, out, lse, B, S, H, scale, none)
                   : fa_fwd<64, false>(stream, qkv, out, lse, B, S, H, scale, none);
}

int attn_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                    void* dqkv, int B, int S, int H, int dh, float scale, const db200_dropout* drop) {
  const db200_dropout none{};
  if (dropout_active(drop))
    return dh == 128 ? fa_bwd<128, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, *drop)
                     : fa_bwd<64, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, *drop);
  return dh == 128 ? fa_bwd<128, false>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none)
                   : fa_bwd<64, false>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none);
}

// sliding window of `radius` keys (radius >= 1); no attention dropout (local layers have none)
int attn_local_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, int dh,
                          int radius, float scale) {
  const db200_dropout none{};
  return dh == 128 ? fa_fwd<128, false, true>(stream, qkv, out, lse, B, S, H, scale, none, radius)
                   : fa_fwd<64, false, true>(stream, qkv, out, lse, B, S, H, scale, none, radius);
}

int attn_local_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                          void* dqkv, int B, int S, int H, int dh, int radius, float scale) {
  const db200_dropout none{};
  return dh == 128 ? fa_bwd<128, false, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none, radius)
                   : fa_bwd<64, false, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none, radius);
}

}  // namespace db200
