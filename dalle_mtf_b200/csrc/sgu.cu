// gMLP token mixing (extension; the spatial gating unit of "Pay Attention to MLPs", DALLE-pytorch's attention type
// 'mlp'): the causal [n, n] mixing products of the training step and the prefill, the SGU's elementwise backward and
// one decoding step.
//
// For every sequence b of n rows (rows b n .. b n + n - 1 of a [B n, C] activation), with W lower triangular:
//   forward  : mixed_b = W gn_b         (M = n positions i, N = C, K = positions j <= i)
//   dgrad    : dgn_b   = W^T dmixed_b   (M = n positions j, N = C, K = positions i >= j)
//   wgrad    : dW     += sum_b dmixed_b gn_b^T over the lower-triangular 128 x 128 tiles (K = (b, channel block))
// One launch each, a persistent warp-specialised wgmma kernel on gemm_common.cuh's tile geometry (BM = 128, BK = 64,
// 128-byte swizzled TMA stages):
//   warp 0     : TMA producer (one elected lane)            smem ring: MX_STAGES x {A 128x64, B 128x64} bf16
//   warps 1-3  : idle (they exit)
//   warps 4-11 : two MMA warpgroups, wgmma m64n128 for rows [64 g, 64 g + 64) of the tile; each runs the epilogue of
//                its half tile straight from the accumulator fragment.
// The tile scheduler walks (m-tile, b, n-tile) for the two sequence products, whose K range ends (forward) or starts
// (dgrad) at the diagonal block, heaviest m-tiles first, and the lower triangle (m-tile, n-tile <= m-tile) for the
// weight gradient.  K blocks past the diagonal inside a tile read W's zero upper triangle, and K blocks past n read
// TMA's zero fill of W, so they add exact zeros.  Every output element is written by one thread once: no atomics.
#include "gemm_common.cuh"
#include "wgmma.cuh"

namespace db200 {

constexpr int MX_BN = 128;
constexpr int MX_STAGES = 5;
constexpr int MX_THREADS = 384;
constexpr uint32_t MX_B_BYTES = MX_BN * BK * 2;
constexpr uint32_t MX_STAGE_BYTES = A_BYTES + MX_B_BYTES;
constexpr size_t MX_SMEM_BYTES = 1024 /*align slack*/ + size_t(MX_STAGES) * MX_STAGE_BYTES + 256 /*barriers*/;
static_assert(MX_SMEM_BYTES <= 227 * 1024, "SGU mixing shared memory exceeds the H100 per-block limit");

constexpr int MX_FWD = 0, MX_DGRAD = 1, MX_WGRAD = 2;

struct MixParams {
  int B, n, C;           // sequences, positions per sequence (= the product's M and, forward / dgrad, its K), channels
  int m_tiles, n_tiles;  // 128-row tiles of n; 128-column tiles of C (forward / dgrad) or of n (wgrad)
  int kb_n;              // 64-wide k-blocks of n (forward / dgrad)
  int c_blocks;          // 64-wide channel blocks of C (wgrad: k-blocks per sequence)
  int total;             // tiles of the launch
  const float* bias;     // forward: c[i], fp32 [n]
  const bf16* res;       // forward: res rows, pitch ldres
  long long ldres;
  bf16* out;             // forward: h; dgrad: dgn ([B n, C] contiguous)
  bf16* mixed;           // forward: bf16(acc + c[i]) for the backward, or NULL
  float* dw;             // wgrad: dW fp32, pitch ldw
  long long ldw;
};

struct MixTile {
  int b, m_blk, n_blk, kb0, kb1;
};

template <int MODE>
__device__ __forceinline__ MixTile mix_tile(const MixParams& p, int tile) {
  MixTile t;
  if constexpr (MODE == MX_WGRAD) {
    // lower triangle in row order: m-tile r holds r + 1 tiles, the first of them at r (r + 1) / 2
    int r = (int)((sqrtf(8.f * tile + 1.f) - 1.f) * 0.5f);
    while ((r + 1) * (r + 2) / 2 <= tile) ++r;
    while (r * (r + 1) / 2 > tile) --r;
    t.m_blk = r;
    t.n_blk = tile - r * (r + 1) / 2;
    t.b = 0;
    t.kb0 = 0;
    t.kb1 = p.B * p.c_blocks;
  } else {
    const int per_m = p.B * p.n_tiles;
    const int mi = tile / per_m;
    const int rem = tile - mi * per_m;
    t.b = rem / p.n_tiles;
    t.n_blk = rem - t.b * p.n_tiles;
    if constexpr (MODE == MX_FWD) {  // K = positions j <= i: the last m-tiles carry the most k-blocks
      t.m_blk = p.m_tiles - 1 - mi;
      t.kb0 = 0;
      t.kb1 = min((t.m_blk * BM + BM) / BK, p.kb_n);
    } else {  // K = positions i >= j: the first m-tiles carry the most
      t.m_blk = mi;
      t.kb0 = t.m_blk * BM / BK;
      t.kb1 = p.kb_n;
    }
  }
  return t;
}

// Operand majors: forward A = W (K-major, row i), B = gn (MN-major); dgrad A = W read MN-major (A[j][i] = W[i][j]),
// B = dmixed (MN-major); wgrad A = dmixed (K-major over channels), B = gn (K-major over channels).
template <int MODE>
__global__ void __launch_bounds__(MX_THREADS, 1)
sgu_mix_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const MixParams p) {
  constexpr int TA = MODE == MX_DGRAD ? 1 : 0;
  constexpr int TB = MODE == MX_WGRAD ? 0 : 1;
  constexpr int STAGES = MX_STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t sA = (raw + 1023u) & ~1023u;  // SWIZZLE_128B tiles need 1024-byte alignment
  const uint32_t sB = sA + STAGES * A_BYTES;
  const uint32_t bars = sA + STAGES * MX_STAGE_BYTES;
  const uint32_t full_bar = bars;                // STAGES x 8 B
  const uint32_t empty_bar = bars + 8 * STAGES;  // STAGES x 8 B

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(full_bar + 8 * i, 1);
      mbar_init(empty_bar + 8 * i, 2);  // one arrive per MMA warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    if (warp != 0) return;
    // ------------------------------------------------------------------ TMA producer
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < p.total; tile += gridDim.x) {
      const MixTile t = mix_tile<MODE>(p, tile);
      const int m0 = t.m_blk * BM, n0 = t.n_blk * MX_BN;
      const int row_b = t.b * p.n;  // first row of sequence b
      for (int kb = t.kb0; kb < t.kb1; ++kb) {
        mbar_wait_mma(empty_bar + 8 * stage, phase ^ 1);
        const uint32_t fb = full_bar + 8 * stage;
        if (elect_one_sync()) {
          mbar_expect_tx(fb, MX_STAGE_BYTES);
          const uint32_t a_dst = sA + stage * A_BYTES;
          const uint32_t b_dst = sB + stage * MX_B_BYTES;
          if constexpr (MODE == MX_WGRAD) {
            const int bs = kb / p.c_blocks;
            const int c0 = (kb - bs * p.c_blocks) * BK;
            tma_load_2d(a_dst, &tmA, fb, c0, bs * p.n + m0);
            tma_load_2d(b_dst, &tmB, fb, c0, bs * p.n + n0);
          } else {
            const int k0 = kb * BK;
            if constexpr (MODE == MX_FWD) {
              tma_load_2d(a_dst, &tmA, fb, k0, m0);
            } else {
#pragma unroll
              for (int s = 0; s < BM / 64; ++s) tma_load_2d(a_dst + s * SLAB_BYTES, &tmA, fb, m0 + 64 * s, k0);
            }
#pragma unroll
            for (int s = 0; s < MX_BN / 64; ++s)
              tma_load_2d(b_dst + s * SLAB_BYTES, &tmB, fb, n0 + 64 * s, row_b + k0);
          }
        }
        __syncwarp();
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }
  // -------------------------------------------------------------------- MMA warpgroups
  const int wg = (warp - 4) >> 2;  // rows [64 wg, 64 wg + 64) of every tile
  constexpr uint64_t astep = TA ? 128u : 2u, bstep = TB ? 128u : 2u;
  const uint32_t a_wg = wg * (TA ? SLAB_BYTES : 64u * 128u);
  float d[MX_BN / 2];
  uint32_t stage = 0, phase = 0;
  const int t128 = threadIdx.x & 127;
  for (int tile = blockIdx.x; tile < p.total; tile += gridDim.x) {
    const MixTile t = mix_tile<MODE>(p, tile);
    uint32_t prev_stage = 0;
#pragma unroll
    for (int i = 0; i < MX_BN / 2; ++i) d[i] = 0.f;
    for (int kb = t.kb0; kb < t.kb1; ++kb) {
      mbar_wait_mma(full_bar + 8 * stage, phase);
      const uint64_t ad0 = smem_desc_sw128(sA + stage * A_BYTES + a_wg, TA ? SLAB_BYTES : 0u, 1024);
      const uint64_t bd0 = smem_desc_sw128(sB + stage * MX_B_BYTES, TB ? SLAB_BYTES : 0u, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) wgmma_m64n128<TA, TB>(d, ad0 + k * astep, bd0 + k * bstep, 1u);
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage goes back to the producer
      if (kb > t.kb0 && t128 == 0) mbar_arrive(empty_bar + 8 * prev_stage);
      prev_stage = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (t128 == 0) mbar_arrive(empty_bar + 8 * prev_stage);

    // fragment of m64n128 (wgmma.cuh, acc_store_smem): d[4 i + 2 h + e] is row r0 + 8 h, column 8 i + c0 + e
    const int r0 = t.m_blk * BM + 64 * wg + 16 * (t128 >> 5) + ((t128 & 31) >> 2);
    const int c0 = t.n_blk * MX_BN + 2 * (t128 & 3);
    if constexpr (MODE == MX_WGRAD) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = r0 + 8 * h;
        if (i >= p.n) continue;
        float* row = p.dw + (long long)i * p.ldw;
#pragma unroll
        for (int q = 0; q < MX_BN / 8; ++q) {
          const int j = c0 + 8 * q;
          // j + 1 <= i keeps both elements in the lower triangle (j even, i integer: j <= i - 1 or j == i)
          if (j > i || j >= p.n) continue;
          if (j + 1 <= i && j + 1 < p.n) {
            float2 v = *reinterpret_cast<float2*>(row + j);
            v.x += d[4 * q + 2 * h];
            v.y += d[4 * q + 2 * h + 1];
            *reinterpret_cast<float2*>(row + j) = v;
          } else {
            row[j] += d[4 * q + 2 * h];
          }
        }
      }
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = r0 + 8 * h;
        if (i >= p.n) continue;
        const long long row = (long long)t.b * p.n + i;
        const float ci = MODE == MX_FWD ? p.bias[i] : 0.f;
#pragma unroll
        for (int q = 0; q < MX_BN / 8; ++q) {
          const int c = c0 + 8 * q;
          if (c >= p.C) continue;
          const float a0 = d[4 * q + 2 * h], a1 = d[4 * q + 2 * h + 1];
          if constexpr (MODE == MX_FWD) {
            const float m0v = a0 + ci, m1v = a1 + ci;
            const float2 r = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.res + row * p.ldres + c));
            *reinterpret_cast<uint32_t*>(p.out + row * p.C + c) = pack_bf16x2(m0v * r.x, m1v * r.y);
            if (p.mixed) *reinterpret_cast<uint32_t*>(p.mixed + row * p.C + c) = pack_bf16x2(m0v, m1v);
          } else {
            *reinterpret_cast<uint32_t*>(p.out + row * p.C + c) = pack_bf16x2(a0, a1);
          }
        }
      }
    }
  }
}

template <int MODE>
static int launch_mix(cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB, const MixParams& p,
                      const char* what) {
  static const cudaError_t attr_rc = cudaFuncSetAttribute(sgu_mix_kernel<MODE>,
                                                          cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                          (int)MX_SMEM_BYTES);  // once, thread-safe (magic static)
  DB200_CUDA(attr_rc);
  const int grid = p.total < sm_count() ? p.total : sm_count();
  sgu_mix_kernel<MODE><<<grid, MX_THREADS, MX_SMEM_BYTES, stream>>>(tmA, tmB, p);
  return check_launch(what);
}

static int mix_geometry(int B, int n, int C, long long ldw, const char* what) {
  DB200_REQUIRE(B > 0 && n > 0 && C > 0, DB200_E_INVALID, "%s: need B, n, C > 0 (got %d, %d, %d)", what, B, n, C);
  DB200_REQUIRE(C % 64 == 0, DB200_E_INVALID, "%s: C %d is not a multiple of 64", what, C);
  DB200_REQUIRE(ldw >= n && ldw % 8 == 0, DB200_E_ALIGN, "%s: ldw %lld must be >= n %d and a multiple of 8", what,
                ldw, n);
  DB200_REQUIRE((long long)B * n <= INT32_MAX, DB200_E_INVALID, "%s: B n = %lld rows exceed 2^31 - 1", what,
                (long long)B * n);
  return DB200_OK;
}

static MixParams mix_params(int B, int n, int C) {
  MixParams p{};
  p.B = B; p.n = n; p.C = C;
  p.m_tiles = (n + BM - 1) / BM;
  p.n_tiles = (C + MX_BN - 1) / MX_BN;
  p.kb_n = (n + BK - 1) / BK;
  p.c_blocks = C / BK;
  p.total = p.m_tiles * B * p.n_tiles;
  return p;
}

// ---------------------------------------------------------------------------------------------------------------------
// SGU backward, one CTA per position i over the rows b n + i of every sequence:
//   dmixed = bf16(dh res),  du_res = bf16(dh mixed gelu'(z_res)),  dc[i] += sum_b sum_c dmixed  (b, then a fixed tree)
// ---------------------------------------------------------------------------------------------------------------------
constexpr int SB_THREADS = 256;

__global__ void __launch_bounds__(SB_THREADS)
sgu_bwd_kernel(const bf16* __restrict__ dh, const bf16* __restrict__ mixed, const bf16* __restrict__ res,
               long long ldres, const bf16* __restrict__ z, long long ldz, bf16* __restrict__ dmixed,
               bf16* __restrict__ du, long long ldu, float* __restrict__ dc, int B, int n, int C) {
  const int i = blockIdx.x;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) {
    const long long row = (long long)b * n + i;
    for (int c = 2 * threadIdx.x; c < C; c += 2 * SB_THREADS) {
      const float2 g = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dh + row * C + c));
      const float2 m = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(mixed + row * C + c));
      const float2 r = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(res + row * ldres + c));
      const float2 zz = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(z + row * ldz + c));
      const uint32_t dm = pack_bf16x2(g.x * r.x, g.y * r.y);
      *reinterpret_cast<uint32_t*>(dmixed + row * C + c) = dm;
      *reinterpret_cast<uint32_t*>(du + row * ldu + c) =
          pack_bf16x2(g.x * m.x * gelu_grad(zz.x), g.y * m.y * gelu_grad(zz.y));
      const float2 dmf = unpack_bf16x2(dm);
      acc += dmf.x;
      acc += dmf.y;
    }
  }
  __shared__ float red[SB_THREADS / 32];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < SB_THREADS / 32; ++w) s += red[w];
    dc[i] += s;
  }
}

// du_gate = bf16(dgate gelu'(z_gate)), rows of C channels
__global__ void __launch_bounds__(256)
sgu_gate_bwd_kernel(const bf16* __restrict__ dg, const bf16* __restrict__ z, long long ldz, bf16* __restrict__ du,
                    long long ldu, long long total2, int C2) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < total2;
       k += (long long)gridDim.x * blockDim.x) {
    const long long row = k / C2;
    const int c = 2 * (int)(k - row * C2);
    const float2 g = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dg + row * (2LL * C2) + c));
    const float2 zz = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(z + row * ldz + c));
    *reinterpret_cast<uint32_t*>(du + row * ldu + c) = pack_bf16x2(g.x * gelu_grad(zz.x), g.y * gelu_grad(zz.y));
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Decoding step at position p for every row r: cache[r][p] = gn[r], then
//   h[r][c] = bf16((sum_{j <= p} W[p][j] cache[r][j][c] + c_sgu[p]) res[r][c]),  the sum in fp32 in j order.
// Grid (C / (2 SD_THREADS) blocks of channel pairs, rows); W's row p is staged in shared memory as fp32.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int SD_THREADS = 128;
constexpr int SD_UNROLL = 8;

__global__ void __launch_bounds__(SD_THREADS)
sgu_decode_kernel(const bf16* __restrict__ gn, const bf16* __restrict__ res, long long ldres,
                  const bf16* __restrict__ w, long long ldw, const float* __restrict__ cbias, bf16* __restrict__ cache,
                  bf16* __restrict__ h, int S, int C, int pos, const int* __restrict__ pos_dev) {
  extern __shared__ float wrow[];
  const int p = pos_dev ? *pos_dev : pos;
  if (p < 0 || p >= S) return;
  for (int j = threadIdx.x; j <= p; j += SD_THREADS) wrow[j] = __bfloat162float(w[(long long)p * ldw + j]);
  __syncthreads();
  const int r = blockIdx.y;
  const int c = 2 * (blockIdx.x * SD_THREADS + threadIdx.x);
  if (c >= C) return;
  bf16* row = cache + (long long)r * S * C + c;
  const uint32_t g = *reinterpret_cast<const uint32_t*>(gn + (long long)r * C + c);
  *reinterpret_cast<uint32_t*>(row + (long long)p * C) = g;
  float a0 = 0.f, a1 = 0.f;
  int j = 0;
  // eight cache rows in flight per step; the sum still adds them one by one in j order
  for (; j + SD_UNROLL <= p; j += SD_UNROLL) {
    uint32_t v[SD_UNROLL];
#pragma unroll
    for (int u = 0; u < SD_UNROLL; ++u) v[u] = __ldcs(reinterpret_cast<const unsigned int*>(row + (long long)(j + u) * C));
#pragma unroll
    for (int u = 0; u < SD_UNROLL; ++u) {
      const float2 f = unpack_bf16x2(v[u]);
      a0 = fmaf(wrow[j + u], f.x, a0);
      a1 = fmaf(wrow[j + u], f.y, a1);
    }
  }
  for (; j < p; ++j) {
    const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(row + (long long)j * C));
    a0 = fmaf(wrow[j], f.x, a0);
    a1 = fmaf(wrow[j], f.y, a1);
  }
  const float2 v = unpack_bf16x2(g);
  a0 = fmaf(wrow[p], v.x, a0);
  a1 = fmaf(wrow[p], v.y, a1);
  const float cb = cbias[p];
  const float2 rr = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(res + (long long)r * ldres + c));
  *reinterpret_cast<uint32_t*>(h + (long long)r * C + c) = pack_bf16x2((a0 + cb) * rr.x, (a1 + cb) * rr.y);
}

// Prefill hand-off: cache[b rep + r][p] = gn[b P + p] for p < P, r < rep (16-byte vectors).
__global__ void __launch_bounds__(256)
sgu_cache_fill_kernel(const uint4* __restrict__ gn, uint4* __restrict__ cache, int P, int S, int rep, int nv,
                      long long total) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < total;
       k += (long long)gridDim.x * blockDim.x) {
    const long long t = k / nv;
    const int v = (int)(k - t * nv);
    const int p = (int)(t % P);
    const long long b = t / P;
    const uint4 val = gn[k];
    for (int r = 0; r < rep; ++r) cache[((b * rep + r) * S + p) * nv + v] = val;
  }
}

static int ew_grid(long long work) {
  const long long cap = (long long)sm_count() * 16;
  const long long blocks = (work + 255) / 256;
  return (int)(blocks < 1 ? 1 : (blocks < cap ? blocks : cap));
}

static bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }

static int sgu_decode_launch(cudaStream_t stream, const void* gn, const void* res, int64_t ldres, const void* w,
                             int64_t ldw, const float* c, void* cache, void* h, int rows, int S, int C, int pos,
                             const int32_t* pos_dev, const char* what) {
  DB200_REQUIRE(gn && res && w && c && cache && h, DB200_E_INVALID, "%s: NULL pointer", what);
  DB200_REQUIRE(rows > 0 && S > 0 && C > 0 && C % 2 == 0 && ldres >= C && ldres % 2 == 0 && ldw >= S, DB200_E_INVALID,
                "%s: need rows, S > 0, even C > 0, even ldres >= C and ldw >= S (got rows=%d S=%d C=%d ldres=%lld "
                "ldw=%lld)", what, rows, S, C, (long long)ldres, (long long)ldw);
  DB200_REQUIRE(S <= 12288, DB200_E_INVALID, "%s: S %d exceeds the 12288 positions staged in shared memory", what, S);
  DB200_REQUIRE(aligned4(gn) && aligned4(res) && aligned4(cache) && aligned4(h), DB200_E_ALIGN,
                "%s: bf16 pairs must be 4-byte aligned", what);
  dim3 grid((C / 2 + SD_THREADS - 1) / SD_THREADS, rows);
  sgu_decode_kernel<<<grid, SD_THREADS, S * sizeof(float), stream>>>(
      static_cast<const bf16*>(gn), static_cast<const bf16*>(res), ldres, static_cast<const bf16*>(w), ldw, c,
      static_cast<bf16*>(cache), static_cast<bf16*>(h), S, C, pos, pos_dev);
  return check_launch(what);
}

}  // namespace db200

using namespace db200;

extern "C" int db200_sgu_mix_fwd(db200_stream_t stream_, const void* w_bf16, int64_t ldw, const void* gn_bf16,
                                 const void* res_bf16, int64_t ldres, const float* c, void* h_bf16, void* mixed_bf16,
                                 int B, int n, int C) {
  const char* what = "sgu_mix_fwd";
  DB200_REQUIRE(w_bf16 && gn_bf16 && res_bf16 && c && h_bf16, DB200_E_INVALID, "%s: NULL pointer", what);
  int rc = mix_geometry(B, n, C, ldw, what);
  if (rc) return rc;
  DB200_REQUIRE(ldres >= C && ldres % 2 == 0 && aligned4(res_bf16) && aligned4(h_bf16) && aligned4(mixed_bf16),
                DB200_E_ALIGN, "%s: res needs an even ldres >= C; res, h and mixed 4-byte alignment", what);
  MixParams p = mix_params(B, n, C);
  p.bias = c;
  p.res = static_cast<const bf16*>(res_bf16);
  p.ldres = ldres;
  p.out = static_cast<bf16*>(h_bf16);
  p.mixed = static_cast<bf16*>(mixed_bf16);
  CUtensorMap tmA, tmB;
  if ((rc = make_tmap_2d(&tmA, w_bf16, (uint64_t)n, (uint64_t)n, (uint64_t)ldw, BK, BM)) != DB200_OK) return rc;
  if ((rc = make_tmap_2d(&tmB, gn_bf16, (uint64_t)C, (uint64_t)B * n, (uint64_t)C, 64, BK)) != DB200_OK) return rc;
  return launch_mix<MX_FWD>(reinterpret_cast<cudaStream_t>(stream_), tmA, tmB, p, what);
}

extern "C" int db200_sgu_mix_dgrad(db200_stream_t stream_, const void* w_bf16, int64_t ldw, const void* dmixed_bf16,
                                   void* dgn_bf16, int B, int n, int C) {
  const char* what = "sgu_mix_dgrad";
  DB200_REQUIRE(w_bf16 && dmixed_bf16 && dgn_bf16, DB200_E_INVALID, "%s: NULL pointer", what);
  int rc = mix_geometry(B, n, C, ldw, what);
  if (rc) return rc;
  DB200_REQUIRE(n % 64 == 0, DB200_E_INVALID, "%s: n %d is not a multiple of 64", what, n);
  MixParams p = mix_params(B, n, C);
  p.out = static_cast<bf16*>(dgn_bf16);
  CUtensorMap tmA, tmB;
  if ((rc = make_tmap_2d(&tmA, w_bf16, (uint64_t)n, (uint64_t)n, (uint64_t)ldw, 64, BK)) != DB200_OK) return rc;
  if ((rc = make_tmap_2d(&tmB, dmixed_bf16, (uint64_t)C, (uint64_t)B * n, (uint64_t)C, 64, BK)) != DB200_OK)
    return rc;
  return launch_mix<MX_DGRAD>(reinterpret_cast<cudaStream_t>(stream_), tmA, tmB, p, what);
}

extern "C" int db200_sgu_mix_wgrad(db200_stream_t stream_, const void* dmixed_bf16, const void* gn_bf16, float* dw,
                                   int64_t ldw, int B, int n, int C) {
  const char* what = "sgu_mix_wgrad";
  DB200_REQUIRE(dmixed_bf16 && gn_bf16 && dw, DB200_E_INVALID, "%s: NULL pointer", what);
  int rc = mix_geometry(B, n, C, ldw, what);
  if (rc) return rc;
  DB200_REQUIRE(n % 64 == 0 && ldw % 2 == 0 && (reinterpret_cast<uintptr_t>(dw) & 7u) == 0, DB200_E_INVALID,
                "%s: n %d must be a multiple of 64 and dW 8-byte aligned", what, n);
  MixParams p = mix_params(B, n, C);
  p.n_tiles = p.m_tiles;
  p.total = p.m_tiles * (p.m_tiles + 1) / 2;
  p.dw = dw;
  p.ldw = ldw;
  CUtensorMap tmA, tmB;
  const uint64_t rows = (uint64_t)B * n;
  if ((rc = make_tmap_2d(&tmA, dmixed_bf16, (uint64_t)C, rows, (uint64_t)C, BK, BM)) != DB200_OK) return rc;
  if ((rc = make_tmap_2d(&tmB, gn_bf16, (uint64_t)C, rows, (uint64_t)C, BK, MX_BN)) != DB200_OK) return rc;
  return launch_mix<MX_WGRAD>(reinterpret_cast<cudaStream_t>(stream_), tmA, tmB, p, what);
}

extern "C" int db200_sgu_bwd(db200_stream_t stream_, const void* dh_bf16, const void* mixed_bf16, const void* res_bf16,
                             int64_t ldres, const void* z_bf16, int64_t ldz, void* dmixed_bf16, void* du_bf16,
                             int64_t ldu, float* dc, int B, int n, int C) {
  DB200_REQUIRE(dh_bf16 && mixed_bf16 && res_bf16 && z_bf16 && dmixed_bf16 && du_bf16 && dc, DB200_E_INVALID,
                "sgu_bwd: NULL pointer");
  DB200_REQUIRE(B > 0 && n > 0 && C > 0 && C % 2 == 0 && ldres >= C && ldz >= C && ldu >= C && ldres % 2 == 0 &&
                    ldz % 2 == 0 && ldu % 2 == 0,
                DB200_E_INVALID, "sgu_bwd: need B, n > 0, even C > 0 and even pitches >= C");
  DB200_REQUIRE(aligned4(dh_bf16) && aligned4(mixed_bf16) && aligned4(res_bf16) && aligned4(z_bf16) &&
                    aligned4(dmixed_bf16) && aligned4(du_bf16),
                DB200_E_ALIGN, "sgu_bwd: bf16 pairs must be 4-byte aligned");
  sgu_bwd_kernel<<<n, SB_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const bf16*>(dh_bf16), static_cast<const bf16*>(mixed_bf16), static_cast<const bf16*>(res_bf16),
      ldres, static_cast<const bf16*>(z_bf16), ldz, static_cast<bf16*>(dmixed_bf16), static_cast<bf16*>(du_bf16), ldu,
      dc, B, n, C);
  return check_launch("sgu_bwd");
}

extern "C" int db200_sgu_gate_bwd(db200_stream_t stream_, const void* dgate_bf16, const void* z_bf16, int64_t ldz,
                                  void* du_bf16, int64_t ldu, int rows, int C) {
  DB200_REQUIRE(dgate_bf16 && z_bf16 && du_bf16, DB200_E_INVALID, "sgu_gate_bwd: NULL pointer");
  DB200_REQUIRE(rows > 0 && C > 0 && C % 2 == 0 && ldz >= C && ldu >= C && ldz % 2 == 0 && ldu % 2 == 0,
                DB200_E_INVALID, "sgu_gate_bwd: need rows > 0, even C > 0 and even pitches >= C");
  DB200_REQUIRE(aligned4(dgate_bf16) && aligned4(z_bf16) && aligned4(du_bf16), DB200_E_ALIGN,
                "sgu_gate_bwd: bf16 pairs must be 4-byte aligned");
  const long long total2 = (long long)rows * (C / 2);
  sgu_gate_bwd_kernel<<<ew_grid(total2), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const bf16*>(dgate_bf16), static_cast<const bf16*>(z_bf16), ldz, static_cast<bf16*>(du_bf16), ldu,
      total2, C / 2);
  return check_launch("sgu_gate_bwd");
}

extern "C" int db200_sgu_decode(db200_stream_t stream_, const void* gn_bf16, const void* res_bf16, int64_t ldres,
                                const void* w_bf16, int64_t ldw, const float* c, void* cache_bf16, void* h_bf16,
                                int rows, int S, int C, int pos) {
  DB200_REQUIRE(pos >= 0 && pos < S, DB200_E_INVALID, "sgu_decode: position %d outside [0, %d)", pos, S);
  return sgu_decode_launch(reinterpret_cast<cudaStream_t>(stream_), gn_bf16, res_bf16, ldres, w_bf16, ldw, c,
                           cache_bf16, h_bf16, rows, S, C, pos, nullptr, "sgu_decode");
}

extern "C" int db200_sgu_decode_dev(db200_stream_t stream_, const void* gn_bf16, const void* res_bf16, int64_t ldres,
                                    const void* w_bf16, int64_t ldw, const float* c, void* cache_bf16, void* h_bf16,
                                    int rows, int S, int C, const int32_t* pos_dev) {
  DB200_REQUIRE(pos_dev, DB200_E_INVALID, "sgu_decode_dev: NULL pos_dev");
  return sgu_decode_launch(reinterpret_cast<cudaStream_t>(stream_), gn_bf16, res_bf16, ldres, w_bf16, ldw, c,
                           cache_bf16, h_bf16, rows, S, C, -1, pos_dev, "sgu_decode_dev");
}

extern "C" int db200_sgu_cache_fill(db200_stream_t stream_, const void* gn_bf16, void* cache_bf16, int B, int P, int C,
                                    int S_cache, int rep) {
  DB200_REQUIRE(gn_bf16 && cache_bf16, DB200_E_INVALID, "sgu_cache_fill: NULL pointer");
  DB200_REQUIRE(B > 0 && P > 0 && C > 0 && C % 8 == 0 && S_cache >= P && rep >= 1, DB200_E_INVALID,
                "sgu_cache_fill: B %d P %d C %d S_cache %d rep %d", B, P, C, S_cache, rep);
  DB200_REQUIRE(aligned16(gn_bf16) && aligned16(cache_bf16), DB200_E_ALIGN,
                "sgu_cache_fill: pointers must be 16-byte aligned");
  const int nv = C / 8;
  const long long total = (long long)B * P * nv;
  sgu_cache_fill_kernel<<<ew_grid(total), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const uint4*>(gn_bf16), static_cast<uint4*>(cache_bf16), P, S_cache, rep, nv, total);
  return check_launch("sgu_cache_fill");
}
