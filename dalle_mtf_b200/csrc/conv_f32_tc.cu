// K11 (fp32 activations) — the discrete-VAE convolutions of an fp32 configuration (vae_example: `bf_16` absent,
// src/vae_tf/models.py:95-109,139-155) on wgmma with fp32-accurate products.
//
// An fp32 value is split into three bf16 parts x = h + m + l (|m| <= 2^-9 |x|, |l| <= 2^-18 |x|, residual <= 2^-27 |x|);
// a product of two split values keeps the six terms down to 2^-18 (hh, hm, mh, hl, lh, mm) — the dropped ones are below
// fp32's own rounding — and all of them accumulate in fp32 registers.  The split happens inside the kernel: the CTA's
// threads read the fp32 pixels / weights from global memory (coalesced, zero-filled outside the image), split them in
// registers and store the three bf16 tiles straight into the 128-byte-swizzled shared-memory layout the wgmma
// descriptors expect; there is no bf16 copy of anything in HBM and no TMA (the producer is the math threads).
// Eight warps = two warpgroups, each of them producer and consumer in turn: store chunk c into one of three smem
// stages, refill the registers with chunk c+2, arrive on the stage's "full" mbarrier, wait for both warpgroups'
// stores, issue the six-product wgmma group for the warpgroup's 64 rows asynchronously, and hand the stage of chunk
// c-1 back ("empty" mbarrier) once its MMAs have retired — the split of chunk c+1 overlaps the MMAs of chunk c.  (In
// the wgrad kernel ptxas currently serialises the wgmma groups (C7518), so there the overlap does not happen.)
//
//   gather-GEMM (forward, conv-transpose forward, both dgrads; the ConvGemmParams of conv.cu):
//       D[128 pixels][64 channels] += A[128 pixels][64 k] * B[64 k][64 channels]      per (tap, 64-channel k chunk)
//   outer product (both wgrads; ConvWgradParams):
//       D[128 a][64 b] += P[64 pixels][128 a]^T * Q[64 pixels][64 b]                  per 64-pixel chunk of one tap
//
// Both operands of the wgrad are "MN-major" tiles (rows = pixels = the contracted index), which is byte for byte the
// same staging as the forward A tile; only the descriptors differ.
#include "common.cuh"
#include "ptx.cuh"
#include "conv_params.cuh"
#include "wgmma.cuh"

namespace db200 {
namespace {

constexpr uint32_t FT_A_PART = 128 * 128;   // [128 rows][64 bf16] or 2 slabs of [64 rows][64 bf16]
constexpr uint32_t FT_B_PART = 64 * 128;    // [64 rows][64 bf16]
constexpr uint32_t FT_STAGE = 3 * FT_A_PART + 3 * FT_B_PART;   // 72 KiB
constexpr int FT_NSTAGE = 3;
constexpr size_t FT_SMEM = 1024 + FT_NSTAGE * FT_STAGE + 64;
static_assert(FT_SMEM <= 227 * 1024, "shared memory exceeds the H100 per-block limit");

__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint4 v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// two floats -> bf16 pairs of the three parts
__device__ __forceinline__ void split3(float a, float b, uint32_t& h, uint32_t& m, uint32_t& l) {
  const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
  const float2 hf = __bfloat1622float2(h2);
  const float ra = a - hf.x, rb = b - hf.y;
  const __nv_bfloat162 m2 = __floats2bfloat162_rn(ra, rb);
  const float2 mf = __bfloat1622float2(m2);
  const __nv_bfloat162 l2 = __floats2bfloat162_rn(ra - mf.x, rb - mf.y);
  h = *reinterpret_cast<const uint32_t*>(&h2);
  m = *reinterpret_cast<const uint32_t*>(&m2);
  l = *reinterpret_cast<const uint32_t*>(&l2);
}

// 8 consecutive floats (two float4) of row `row`, 16-byte segment `seg` -> the three swizzled tiles at base, +part, +2 part
__device__ __forceinline__ void stage8(uint32_t base, uint32_t part, uint32_t row, uint32_t seg, float4 v0, float4 v1) {
  uint4 h, m, l;
  split3(v0.x, v0.y, h.x, m.x, l.x);
  split3(v0.z, v0.w, h.y, m.y, l.y);
  split3(v1.x, v1.y, h.z, m.z, l.z);
  split3(v1.z, v1.w, h.w, m.w, l.w);
  const uint32_t off = row * 128u + (((seg ^ (row & 7u)) & 7u) << 4);
  st_shared_v4(base + off, h);
  st_shared_v4(base + part + off, m);
  st_shared_v4(base + 2 * part + off, l);
}

// the six products with weight >= 2^-18, smallest first (m64 x 64 x 16 each, this warpgroup's 64 rows)
template <int TA, int TB>
__device__ __forceinline__ void mma6(float* d, const uint64_t (&ad)[3], const uint64_t (&bd)[3], uint64_t astep,
                                     uint64_t bstep, bool first) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint64_t a0 = ad[0] + kk * astep, a1 = ad[1] + kk * astep, a2 = ad[2] + kk * astep;
    const uint64_t b0 = bd[0] + kk * bstep, b1 = bd[1] + kk * bstep, b2 = bd[2] + kk * bstep;
    wgmma_m64n64<TA, TB>(d, a1, b1, (first && kk == 0) ? 0u : 1u);
    wgmma_m64n64<TA, TB>(d, a0, b2, 1u);
    wgmma_m64n64<TA, TB>(d, a2, b0, 1u);
    wgmma_m64n64<TA, TB>(d, a0, b1, 1u);
    wgmma_m64n64<TA, TB>(d, a1, b0, 1u);
    wgmma_m64n64<TA, TB>(d, a0, b0, 1u);
  }
}

constexpr int FT_THREADS = 256;   // two warpgroups: producers and wgmma consumers in turn
struct FtSmem {
  uint32_t stage0;     // stage s at stage0 + s * FT_STAGE: A parts first, B parts at + 3 * FT_A_PART
  uint32_t bar0;       // bar0 + 8 s: "the MMAs that read stage s have retired";  bar0 + 8 (3 + s): "stage s is written"
  __device__ __forceinline__ uint32_t stage(int s) const { return stage0 + s * FT_STAGE; }
  __device__ __forceinline__ uint32_t bar(int s) const { return bar0 + 8 * s; }
  __device__ __forceinline__ uint32_t full(int s) const { return bar0 + 8 * (FT_NSTAGE + s); }
};

__device__ __forceinline__ FtSmem ft_carve(uint8_t* raw_ptr) {
  const uint32_t raw = smem_u32(raw_ptr);
  const uint32_t base = (raw + 1023u) & ~1023u;
  FtSmem s;
  s.stage0 = base;
  s.bar0 = base + FT_NSTAGE * FT_STAGE;
  return s;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// gather-GEMM
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FT_THREADS)
conv_gemm_f32_tc_kernel(const ConvGemmParams p) {
  extern __shared__ uint8_t ft_smem_raw[];
  const FtSmem sm = ft_carve(ft_smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const long long M = (long long)p.NB * p.OH * p.OW;
  const long long m0 = (long long)blockIdx.x * 128;
  const int n0 = blockIdx.y * 64;
  const float* x = reinterpret_cast<const float*>(p.x);

  if (tid == 0) {
    for (int i = 0; i < FT_NSTAGE; ++i) { mbar_init(sm.bar(i), 2); mbar_init(sm.full(i), 8); }
    fence_mbar_init();
  }
  __syncthreads();

  // A loader: pixel row (tid >> 1), channels (tid & 1) * 32 .. + 31 of the chunk
  const uint32_t a_row = tid >> 1, a_seg0 = (tid & 1) * 4;
  const long long am = m0 + a_row;
  const bool a_ok = am < M;
  int a_n = 0, a_oy = 0, a_ox = 0;
  if (a_ok) {
    a_ox = (int)(am % p.OW);
    a_oy = (int)((am / p.OW) % p.OH);
    a_n = (int)(am / ((long long)p.OW * p.OH));
  }
  // B loader: 64 rows x 64 contiguous elements; rows run along k when the channels produced are contiguous in memory
  // (MN-major B tile), along n when the contracted channels are (K-major B tile)
  const bool b_mn = (p.w_n_stride == 1);
  const uint32_t b_row = tid >> 2, b_seg0 = (tid & 3) * 2;
  const int kch = p.K >> 6;
  const int nchunk = p.ntaps * kch;

  auto load_chunk = [&](int c, float4 (&ra)[8], float4 (&rb)[4]) {
    const int t = c / kch, k0 = (c - t * kch) << 6;
    const int iy = a_oy * p.in_stride + p.taps[t].dy, ix = a_ox * p.in_stride + p.taps[t].dx;
    const bool ok = a_ok && iy >= 0 && iy < p.in_H && ix >= 0 && ix < p.in_W;
    if (ok) {
      const float4* src = reinterpret_cast<const float4*>(x + (((long long)a_n * p.in_H + iy) * p.in_W + ix) * p.K + k0 +
                                                          a_seg0 * 8);
#pragma unroll
      for (int j = 0; j < 8; ++j) ra[j] = __ldg(src + j);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) ra[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const float* wt = p.w + p.taps[t].w_off;
    const float4* wsrc =
        b_mn ? reinterpret_cast<const float4*>(wt + (long long)(k0 + b_row) * p.w_k_stride + n0 + b_seg0 * 8)
             : reinterpret_cast<const float4*>(wt + (long long)(n0 + b_row) * p.w_n_stride + k0 + b_seg0 * 8);
#pragma unroll
    for (int j = 0; j < 4; ++j) rb[j] = __ldg(wsrc + j);
  };
  auto store_chunk = [&](int s, const float4 (&ra)[8], const float4 (&rb)[4]) {
    const uint32_t sA = sm.stage(s), sB = sm.stage(s) + 3 * FT_A_PART;
#pragma unroll
    for (int j = 0; j < 4; ++j) stage8(sA, FT_A_PART, a_row, a_seg0 + j, ra[2 * j], ra[2 * j + 1]);
#pragma unroll
    for (int j = 0; j < 2; ++j) stage8(sB, FT_B_PART, b_row, b_seg0 + j, rb[2 * j], rb[2 * j + 1]);
  };

  // chunk c: registers -> stage c % 3 (once the MMAs of chunk c-3 have read it), refill the register set with chunk
  // c+2, publish, wait for the other warpgroup's half, issue this warpgroup's six-product group (rows 64 wg ..)
  float d[32];
  auto do_chunk = [&](int c, float4 (&ra)[8], float4 (&rb)[4]) {
    const int s = c % FT_NSTAGE;
    if (c >= FT_NSTAGE) mbar_wait_mma(sm.bar(s), (uint32_t)((c / FT_NSTAGE - 1) & 1));
    store_chunk(s, ra, rb);
    if (c + 2 < nchunk) load_chunk(c + 2, ra, rb);
    fence_proxy_async_smem();   // generic-proxy stores -> visible to wgmma (async proxy)
    __syncwarp();
    if (lane == 0) mbar_arrive(sm.full(s));
    mbar_wait_mma(sm.full(s), (uint32_t)((c / FT_NSTAGE) & 1));
    const uint32_t sA = sm.stage(s) + wg * (64u * 128u), sB = sm.stage(s) + 3 * FT_A_PART;
    uint64_t ad[3], bd[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      ad[i] = smem_desc_sw128(sA + i * FT_A_PART, 0, 1024);
      bd[i] = smem_desc_sw128(sB + i * FT_B_PART, b_mn ? FT_B_PART : 0u, 1024);
    }
    wgmma_fence();
    if (b_mn) mma6<0, 1>(d, ad, bd, 2u, 128u, c == 0);
    else      mma6<0, 0>(d, ad, bd, 2u, 2u, c == 0);
    wgmma_commit();
    wgmma_wait<1>();   // chunk c-1 has retired: its stage may be overwritten
    if (c > 0 && (tid & 127) == 0) mbar_arrive(sm.bar((c - 1) % FT_NSTAGE));
  };
  {
    float4 ra0[8], rb0[4], ra1[8], rb1[4];
    load_chunk(0, ra0, rb0);
    if (nchunk > 1) load_chunk(1, ra1, rb1);
    for (int c = 0; c < nchunk; c += 2) {
      do_chunk(c, ra0, rb0);
      if (c + 1 < nchunk) do_chunk(c + 1, ra1, rb1);
    }
    wgmma_wait<0>();
    __syncthreads();   // every MMA has read its stage: stage 0 holds the accumulator tile from here on
    acc_store_smem<64>(d, sm.stage(0) >> 2, 64 * wg);
    __syncthreads();
  }

  // ---- epilogue: warp w reads accumulator rows 32 (w & 3) .., columns 32 (w >> 2) ..; one pixel x 32 channels per thread
  {
    const int q = warp & 3, half = warp >> 2;
    const long long m = m0 + q * 32 + lane;
    uint32_t r[32];
    acc_ld_x32((sm.stage(0) >> 2) + (q * 32 + lane) * 64 + half * 32, r);
    if (m < M) {
      const int ox = (int)(m % p.OW);
      const int oy = (int)((m / p.OW) % p.OH);
      const int n = (int)(m / ((long long)p.OW * p.OH));
      const long long o =
          (((long long)n * p.out_H + (oy * p.out_stride + p.oa)) * p.out_W + (ox * p.out_stride + p.ob)) * p.Nn + n0 +
          half * 32;
      float* y = reinterpret_cast<float*>(p.y) + o;
      const float* res = p.residual ? reinterpret_cast<const float*>(p.residual) + o : nullptr;
      const float* msk = p.mask ? reinterpret_cast<const float*>(p.mask) + o : nullptr;
      const float* bias = p.bias ? p.bias + n0 + half * 32 : nullptr;
#pragma unroll
      for (int e = 0; e < 32; e += 4) {
        float v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = __uint_as_float(r[e + u]);
        if (bias) {
          const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + e));
          v[0] += b4.x; v[1] += b4.y; v[2] += b4.z; v[3] += b4.w;
        }
        if (p.relu) {
#pragma unroll
          for (int u = 0; u < 4; ++u) v[u] = fmaxf(v[u], 0.f);
        }
        if (msk) {
          const float4 m4 = *reinterpret_cast<const float4*>(msk + e);
          v[0] = m4.x > 0.f ? v[0] : 0.f; v[1] = m4.y > 0.f ? v[1] : 0.f;
          v[2] = m4.z > 0.f ? v[2] : 0.f; v[3] = m4.w > 0.f ? v[3] : 0.f;
        }
        if (res) {
          const float4 r4 = *reinterpret_cast<const float4*>(res + e);
          v[0] += r4.x; v[1] += r4.y; v[2] += r4.z; v[3] += r4.w;
        }
        *reinterpret_cast<float4*>(y + e) = make_float4(v[0], v[1], v[2], v[3]);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// outer product (wgrad): CTA = (128 a-channels, 64 b-channels, one tap, one pixel range); red.add into dw
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FT_THREADS)
conv_wgrad_f32_tc_kernel(const ConvWgradParams p) {
  extern __shared__ uint8_t ft_smem_raw[];
  const FtSmem sm = ft_carve(ft_smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int a0 = blockIdx.x * 128, b0 = blockIdx.y * 64;
  const int t = blockIdx.z % p.ntaps, split = blockIdx.z / p.ntaps;
  const long long M = (long long)p.NB * p.OH * p.OW;
  const long long per = ((M + p.splits - 1) / p.splits + 63) / 64 * 64;
  const long long mbeg = split * per, mend = (mbeg + per < M) ? mbeg + per : M;
  const float* P = reinterpret_cast<const float*>(p.P);
  const float* Q = reinterpret_cast<const float*>(p.Q);
  const WgradTap tap = p.taps[t];

  if (tid == 0) {
    for (int i = 0; i < FT_NSTAGE; ++i) { mbar_init(sm.bar(i), 2); mbar_init(sm.full(i), 8); }
    fence_mbar_init();
  }
  __syncthreads();
  const int nchunk = mbeg < mend ? (int)((mend - mbeg + 63) / 64) : 0;

  // loader: pixel row (tid >> 2) of the 64-pixel chunk; P channels a0 + (tid & 3) * 32 .. + 31 (slab (tid & 3) >> 1),
  // Q channels b0 + (tid & 3) * 16 .. + 15
  const uint32_t row = tid >> 2, pq = tid & 3;
  const uint32_t p_slab = pq >> 1, p_seg0 = (pq & 1) * 4, q_seg0 = pq * 2;
  const bool pa_ok = a0 + (int)pq * 32 < p.pC;   // pC is a multiple of 64: a whole 32-channel run is in or out

  auto load_chunk = [&](int c, float4 (&rp)[8], float4 (&rq)[4]) {
    const long long m = mbeg + (long long)c * 64 + row;
    bool pok = false, qok = false;
    const float *psrc = P, *qsrc = Q;
    if (m < mend) {
      const int ox = (int)(m % p.OW);
      const int oy = (int)((m / p.OW) % p.OH);
      const int n = (int)(m / ((long long)p.OW * p.OH));
      const int py = oy * p.p_stride + tap.pdy, px = ox * p.p_stride + tap.pdx;
      const int qy = oy * p.q_stride + tap.qdy, qx = ox * p.q_stride + tap.qdx;
      pok = pa_ok && py >= 0 && py < p.pH && px >= 0 && px < p.pW;
      qok = qy >= 0 && qy < p.qH && qx >= 0 && qx < p.qW;
      psrc = P + (((long long)n * p.pH + py) * p.pW + px) * p.pC + a0 + pq * 32;
      qsrc = Q + (((long long)n * p.qH + qy) * p.qW + qx) * p.qC + b0 + pq * 16;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) rp[j] = pok ? __ldg(reinterpret_cast<const float4*>(psrc) + j) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 4; ++j) rq[j] = qok ? __ldg(reinterpret_cast<const float4*>(qsrc) + j) : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  auto store_chunk = [&](int s, const float4 (&rp)[8], const float4 (&rq)[4]) {
    const uint32_t sA = sm.stage(s) + p_slab * FT_B_PART, sB = sm.stage(s) + 3 * FT_A_PART;
#pragma unroll
    for (int j = 0; j < 4; ++j) stage8(sA, FT_A_PART, row, p_seg0 + j, rp[2 * j], rp[2 * j + 1]);
#pragma unroll
    for (int j = 0; j < 2; ++j) stage8(sB, FT_B_PART, row, q_seg0 + j, rq[2 * j], rq[2 * j + 1]);
  };

  // both operands MN-major (K = pixels); warpgroup wg takes the 64-channel slab wg of P (accumulator rows 64 wg ..)
  float d[32];
  auto do_chunk = [&](int c, float4 (&rp)[8], float4 (&rq)[4]) {
    const int s = c % FT_NSTAGE;
    if (c >= FT_NSTAGE) mbar_wait_mma(sm.bar(s), (uint32_t)((c / FT_NSTAGE - 1) & 1));
    store_chunk(s, rp, rq);
    if (c + 2 < nchunk) load_chunk(c + 2, rp, rq);
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) mbar_arrive(sm.full(s));
    mbar_wait_mma(sm.full(s), (uint32_t)((c / FT_NSTAGE) & 1));
    const uint32_t sA = sm.stage(s) + wg * FT_B_PART, sB = sm.stage(s) + 3 * FT_A_PART;
    uint64_t ad[3], bd[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      ad[i] = smem_desc_sw128(sA + i * FT_A_PART, FT_B_PART, 1024);
      bd[i] = smem_desc_sw128(sB + i * FT_B_PART, FT_B_PART, 1024);
    }
    wgmma_fence();
    mma6<1, 1>(d, ad, bd, 128u, 128u, c == 0);    // 16 pixels = 16 rows x 128 B = 2 KiB per K-step
    wgmma_commit();
    wgmma_wait<1>();
    if (c > 0 && (tid & 127) == 0) mbar_arrive(sm.bar((c - 1) % FT_NSTAGE));
  };
  if (nchunk == 0) return;  // uniform across the CTA
  {
    float4 rp0[8], rq0[4], rp1[8], rq1[4];
    load_chunk(0, rp0, rq0);
    if (nchunk > 1) load_chunk(1, rp1, rq1);
    for (int c = 0; c < nchunk; c += 2) {
      do_chunk(c, rp0, rq0);
      if (c + 1 < nchunk) do_chunk(c + 1, rp1, rq1);
    }
    wgmma_wait<0>();
    __syncthreads();   // every MMA has read its stage: stage 0 holds the accumulator tile from here on
    acc_store_smem<64>(d, sm.stage(0) >> 2, 64 * wg);
    __syncthreads();
    const int q = warp & 3, half = warp >> 2;
    const int a = a0 + q * 32 + lane;
    uint32_t r[32];
    acc_ld_x32((sm.stage(0) >> 2) + (q * 32 + lane) * 64 + half * 32, r);
    if (a < p.pC) {
      float* dw = p.dw + tap.w_off + (long long)a * p.a_stride + (long long)(b0 + half * 32) * p.b_stride;
#pragma unroll
      for (int e = 0; e < 32; ++e) atomicAdd(dw + (long long)e * p.b_stride, __uint_as_float(r[e]));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------

bool conv_gemm_f32_tc_ok(const ConvGemmParams& p) {
  if (p.K < 64 || (p.K & 63) || p.Nn < 64 || (p.Nn & 63)) return false;
  if (!(p.w_n_stride == 1 || p.w_k_stride == 1)) return false;
  if ((p.w_n_stride == 1 ? p.w_k_stride : p.w_n_stride) & 3) return false;
  for (int t = 0; t < p.ntaps; ++t)
    if (p.taps[t].w_off & 3) return false;
  return aligned16(p.x) && aligned16(p.w) && aligned16(p.y) && (!p.bias || aligned16(p.bias)) &&
         (!p.residual || aligned16(p.residual)) && (!p.mask || aligned16(p.mask));
}

int conv_gemm_f32_tc_launch(cudaStream_t stream, const ConvGemmParams& p) {
  static const cudaError_t attr_rc = cudaFuncSetAttribute(conv_gemm_f32_tc_kernel,
                                                          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FT_SMEM);
  DB200_CUDA(attr_rc);
  const long long M = (long long)p.NB * p.OH * p.OW;
  dim3 grid((unsigned)((M + 127) / 128), (unsigned)(p.Nn / 64));
  conv_gemm_f32_tc_kernel<<<grid, FT_THREADS, FT_SMEM, stream>>>(p);
  return check_launch("conv_gemm_f32_tc_kernel");
}

bool conv_wgrad_f32_tc_ok(const ConvWgradParams& p) {
  if (p.pC < 64 || (p.pC & 63) || p.qC < 64 || (p.qC & 63)) return false;
  return aligned16(p.P) && aligned16(p.Q);
}

int conv_wgrad_f32_tc_launch(cudaStream_t stream, ConvWgradParams& p) {
  static const cudaError_t attr_rc = cudaFuncSetAttribute(conv_wgrad_f32_tc_kernel,
                                                          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FT_SMEM);
  DB200_CUDA(attr_rc);
  const long long M = (long long)p.NB * p.OH * p.OW;
  const int tiles = ((p.pC + 127) / 128) * (p.qC / 64) * p.ntaps;
  int splits = (sm_count() * 2 + tiles - 1) / tiles;
  const long long max_splits = (M + 255) / 256;   // at least four 64-pixel chunks per CTA
  if (splits > max_splits) splits = (int)max_splits;
  if (splits < 1) splits = 1;
  p.splits = splits;
  dim3 grid((p.pC + 127) / 128, p.qC / 64, p.ntaps * splits);
  conv_wgrad_f32_tc_kernel<<<grid, FT_THREADS, FT_SMEM, stream>>>(p);
  return check_launch("conv_wgrad_f32_tc_kernel");
}

}  // namespace db200
