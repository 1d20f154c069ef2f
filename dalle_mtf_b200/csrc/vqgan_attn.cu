// K14 long — the AttnBlock's non-causal single-head attention over S > 256 positions at C = 512 (the 32 x 32 grids of
// a Gumbel f8 VQGAN and of an f16 model's mid block at 512 px), on wgmma.  o_i = sum_j softmax_j(scale q_i . k_j) v_j.
//
// One CTA = (image b, 64 queries) = two warpgroups.  The Q tile stays in shared memory; K and V are visited in 64-row
// tiles, in key order, each loaded once with cp.async into the 128B-swizzled [8 atoms][64 rows][64 bf16] layout of
// the wgmma descriptors and multiplied synchronously (no pipelining).  Per key tile:
//   1. warpgroup w multiplies Q[:, 256 w .. + 256) K[:, 256 w .. + 256)^T into a 64 x 64 fp32 partial score tile;
//      the two partials are exchanged through shared memory and added (a + b == b + a in IEEE arithmetic, so both
//      warpgroups hold the same scores bit for bit and run the same online softmax);
//   2. an fp32 online softmax in the exp2 domain rescales the running row sums and accumulators;
//   3. P is packed to bf16 in registers (as K4 does) and warpgroup w adds P V[:, 256 w .. + 256) into its 64 x 256
//      fp32 accumulator.
// No atomics and a fixed key order: the result is bit-reproducible and an image's output does not depend on B.
#include "gemm_common.cuh"  // cp.async helpers, kLog2e
#include "wgmma.cuh"

namespace db200 {
namespace {

constexpr int AL_ROWS = 64;                            // queries per CTA, keys per tile
constexpr int AL_C = 512;                              // the one width the kernel covers
constexpr int AL_THREADS = 256;                        // two warpgroups
constexpr int AL_LD = 3 * AL_C;                        // qkv row stride (q | k | v)
constexpr int AL_SMIN = 256, AL_SMAX = 4096;           // S range: 256 < S <= 4096 (S <= 256 is K14's)
constexpr uint32_t AL_TILE = AL_ROWS * AL_C * 2;       // 64 KiB bf16 tile
constexpr uint32_t AL_XCH = AL_ROWS * AL_ROWS * 4;     // 16 KiB fp32 partial score tile per warpgroup
constexpr size_t AL_SMEM = 1024 + 3 * (size_t)AL_TILE + 2 * AL_XCH;

// rows [0, 64) x 512 bf16 at src (row stride 3 C) -> swizzled tile at dst; the caller commits.  Thread tid copies
// column chunk c = tid % 64 of rows tid / 64 + 4 i, so one source pointer with constant offsets serves all 16 copies.
__device__ __forceinline__ void al_load_tile(uint32_t dst, const bf16* src, int tid) {
  constexpr int CPR = AL_C / 8;  // 16-byte chunks per row
  const int r0 = tid / CPR, c = tid % CPR;
  const bf16* p = src + r0 * AL_LD + c * 8;
  const uint32_t d = dst + (c >> 3) * (AL_ROWS * 128) + r0 * 128;
#pragma unroll
  for (int i = 0; i < AL_ROWS * CPR / AL_THREADS; ++i) {
    const int r = r0 + 4 * i;
    cp_async16_zfill(d + 512 * i + ((((c & 7) ^ (r & 7)) & 7) << 4), p + 4 * i * AL_LD, true);
  }
}
// K-major descriptor of k-step ks (16 channels) of a tile: 64-channel atoms 8 KiB apart
__device__ __forceinline__ uint64_t al_kdesc(uint32_t tile, int ks) {
  return smem_desc_sw128(tile + (ks >> 2) * (AL_ROWS * 128) + (ks & 3) * 32, 0, 1024);
}
// MN-major descriptor of k-step ks (16 key rows) of the tile's 128 columns from atom `atom` on (B operand, N = 128)
__device__ __forceinline__ uint64_t al_ndesc(uint32_t tile, int atom, int ks) {
  return smem_desc_sw128(tile + atom * (AL_ROWS * 128) + ks * 2048, AL_ROWS * 128, 1024);
}
__device__ __forceinline__ float al_quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float al_quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

}  // namespace

// grid (S / 64, B), 256 threads.  Fragment of m64nNk16 (wgmma.cuh): thread t of a warpgroup holds rows
// fr = 16 (t / 32) + (t % 32) / 4 and fr + 8, columns 8 i + 2 (t % 4) + {0, 1}.
__global__ void __launch_bounds__(AL_THREADS, 1)
attn_noncausal_long_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ out, int S, float scale) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base, sK = base + AL_TILE, sV = base + 2 * AL_TILE, sX = base + 3 * AL_TILE;
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int fr = 16 * (t >> 5) + ((t & 31) >> 2), fc = 2 * (t & 3);
  const int q0 = blockIdx.x * AL_ROWS, b = blockIdx.y;
  const bf16* X = qkv + (long long)b * S * AL_LD;
  const float sl2 = scale * kLog2e;
  // this warpgroup's exchange slot and the other's: float4 j of thread t at word 4 (128 j + t)
  const uint32_t x_mine = sX + wg * AL_XCH + t * 16, x_other = sX + (wg ^ 1) * AL_XCH + t * 16;

  al_load_tile(sQ, X + (long long)q0 * AL_LD, threadIdx.x);
  float o[128], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 128; ++i) o[i] = 0.f;

  for (int k0 = 0; k0 < S; k0 += AL_ROWS) {
    // Opaque copies of the loop-invariant addresses: the tile-load offsets and the 40 wgmma descriptors are recomputed
    // per tile instead of being hoisted out of the loop into registers the 128 accumulators need.
    uint32_t q_s = sQ, k_s = sK, v_s = sV;
    int tid = threadIdx.x;
    asm volatile("" : "+r"(q_s), "+r"(k_s), "+r"(v_s), "+r"(tid));
    __syncthreads();  // the previous tile's K / V and exchanged scores are no longer read
    al_load_tile(k_s, X + (long long)k0 * AL_LD + AL_C, tid);
    al_load_tile(v_s, X + (long long)k0 * AL_LD + 2 * AL_C, tid);
    cp_async_commit();
    cp_async_wait<0>();
    fence_proxy_async_smem();
    __syncthreads();

    float s[32];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 16; ++ks)
      wgmma_m64n64<0, 0>(s, al_kdesc(q_s, 16 * wg + ks), al_kdesc(k_s, 16 * wg + ks), ks > 0);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < 8; ++j)
      asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(x_mine + j * 2048), "f"(s[4 * j]),
                   "f"(s[4 * j + 1]), "f"(s[4 * j + 2]), "f"(s[4 * j + 3])
                   : "memory");
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float r0, r1, r2, r3;
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                   : "=f"(r0), "=f"(r1), "=f"(r2), "=f"(r3)
                   : "r"(x_other + j * 2048)
                   : "memory");
      s[4 * j] += r0; s[4 * j + 1] += r1; s[4 * j + 2] += r2; s[4 * j + 3] += r3;
    }

    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      s[i] *= sl2;
      mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
    }
    float alpha[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const float mn = fmaxf(m[hh], al_quad_max(mx[hh]));
      alpha[hh] = exp2f(m[hh] - mn);
      m[hh] = mn;
      l[hh] *= alpha[hh];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      o[4 * i + 0] *= alpha[0]; o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      s[i] = exp2f(s[i] - m[(i >> 1) & 1]);
      l[(i >> 1) & 1] += s[i];
    }
    uint32_t a[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      a[ks][0] = pack_bf16x2(s[8 * ks + 0], s[8 * ks + 1]);
      a[ks][1] = pack_bf16x2(s[8 * ks + 2], s[8 * ks + 3]);
      a[ks][2] = pack_bf16x2(s[8 * ks + 4], s[8 * ks + 5]);
      a[ks][3] = pack_bf16x2(s[8 * ks + 6], s[8 * ks + 7]);
    }
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      wgmma_rs_m64n128<1>(o, a[ks], al_ndesc(v_s, 4 * wg, ks), 1u);
      wgmma_rs_m64n128<1>(o + 64, a[ks], al_ndesc(v_s, 4 * wg + 2, ks), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
  }

  float inv[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) inv[hh] = 1.f / al_quad_sum(l[hh]);
  // o[4 i + ...] holds column 8 i + fc of this warpgroup's 256 (i >= 16: the second n128 product's 8 (i - 16) + fc)
  bf16* dst = out + ((long long)b * S + q0) * AL_C + 256 * wg + fc;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    bf16* d = dst + (long long)(fr + 8 * hh) * AL_C;
#pragma unroll
    for (int i = 0; i < 32; ++i)
      *reinterpret_cast<uint32_t*>(d + 8 * i) =
          pack_bf16x2(o[4 * i + 2 * hh] * inv[hh], o[4 * i + 2 * hh + 1] * inv[hh]);
  }
}

}  // namespace db200

using namespace db200;

extern "C" int db200_attn_noncausal_long_fwd(db200_stream_t stream_, const void* qkv, void* out, int B, int S, int C,
                                             float scale) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(qkv && out && B > 0 && S > 0 && C > 0, DB200_E_INVALID, "attn_noncausal_long_fwd: bad arguments");
  DB200_REQUIRE(C == AL_C && S % AL_ROWS == 0 && S > AL_SMIN && S <= AL_SMAX && B <= 65535, DB200_E_UNSUPPORTED,
                "attn_noncausal_long_fwd: C = %d must be %d, S = %d a multiple of %d with %d < S <= %d, and B = %d "
                "at most 65535",
                C, AL_C, S, AL_ROWS, AL_SMIN, AL_SMAX, B);
  DB200_REQUIRE(aligned16(qkv) && aligned16(out), DB200_E_ALIGN,
                "attn_noncausal_long_fwd: pointers must be 16-byte aligned");
  DB200_CUDA(cudaFuncSetAttribute(attn_noncausal_long_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)AL_SMEM));
  attn_noncausal_long_kernel<<<dim3(S / AL_ROWS, B), AL_THREADS, AL_SMEM, stream>>>(
      reinterpret_cast<const bf16*>(qkv), reinterpret_cast<bf16*>(out), S, scale);
  return check_launch("attn_noncausal_long_kernel");
}
