// K11 (first layer) — the 4x4 / stride-2 / SAME convolution of the RGB image (Cin = 3) on wgmma.
//
// Reference: the first conv_downsample of DiscreteVAE.encoder, src/vae_tf/models.py:95 (tf.layers.conv2d, HWIO kernel).
// K = 4*4*3 = 48 is too thin for a TMA-fed implicit GEMM (a 3-channel pixel is 12 bytes), so the CTA gathers the
// patches itself: a 128-pixel output tile (8 x 16) is staged as an A operand [128 pixels][64] (48 taps + 16 zero columns)
// in the 128-byte-swizzled K-major layout the wgmma descriptor expects, the weights as B [Cout][64] likewise, and the
// CTA's warpgroup produces the tile in 64 x 64 blocks (wgmma m64n64k16, K = 64) in registers.  The fp32 pixels are split
// into bf16 hi + lo parts (two A tiles, two accumulating MMA groups), so the input keeps ~16 bits of mantissa; the
// weights are rounded to bf16 like those of every other tensor-core layer.  Output: bias added in fp32, rounded to
// bf16, NHWC, straight from the accumulator fragment.  Also absorbs the fp32 -> bf16 cast of the image.  HBM-bound by
// design: 12 B read + 2*Cout B written per output pixel.
#include "common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace db200 {
namespace {

constexpr int CFT_TH = 8, CFT_TW = 16;                    // output tile (128 pixels = accumulator rows)
constexpr int CFT_PH = 2 * CFT_TH + 2, CFT_PW = 2 * CFT_TW + 2;
constexpr uint32_t CFT_A_BYTES = 128 * 128;               // [128][64] bf16
constexpr uint32_t CFT_PATCH_FLOATS = CFT_PH * CFT_PW * 3;

__device__ __forceinline__ void st_shared_v4u(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

}  // namespace

// smem: [1024 align] A_hi | A_lo | B [Cout][64] bf16 | patch f32 [PH][PW][3] | bias f32 [Cout]
__global__ void __launch_bounds__(128)
conv_first_tc_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                     bf16* __restrict__ y, int NB, int H, int W, int Cout) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t sAh = base, sAl = sAh + CFT_A_BYTES, sB = sAl + CFT_A_BYTES;
  const uint32_t sPatch = sB + Cout * 128;
  const uint32_t sBias = sPatch + CFT_PATCH_FLOATS * 4;
  float* patch = reinterpret_cast<float*>(smem_raw + (sPatch - raw));
  float* sbias = reinterpret_cast<float*>(smem_raw + (sBias - raw));

  const int tid = threadIdx.x, warp = tid >> 5;
  const int Ho = H / 2, Wo = W / 2;
  const int tiles_w = (Wo + CFT_TW - 1) / CFT_TW, tiles_h = (Ho + CFT_TH - 1) / CFT_TH;
  const int n_tiles = tiles_w * tiles_h * NB;

  // ---- once per CTA: weights -> B[n][k] = bf16(w[k][n]) (k < 48; zero beyond), swizzled K-major; bias
  for (int i = tid; i < Cout * 8; i += 128) {  // (row n, 16-byte chunk j of 8 taps)
    const int n = i >> 3, j = i & 7;
    uint32_t pk[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k0 = j * 8 + 2 * e;
      const float a = (k0 < 48) ? w[(long long)k0 * Cout + n] : 0.f;
      const float b = (k0 + 1 < 48) ? w[(long long)(k0 + 1) * Cout + n] : 0.f;
      pk[e] = pack_bf16x2(a, b);
    }
    st_shared_v4u(sB + n * 128 + (((j ^ (n & 7)) & 7) << 4), pk[0], pk[1], pk[2], pk[3]);
  }
  for (int i = tid; i < Cout; i += 128) sbias[i] = bias ? bias[i] : 0.f;
  __syncthreads();
  const int ly = tid / CFT_TW, lx = tid % CFT_TW;
  // accumulator fragment of m64n64: rows 16 warp + lane/4 (+8), columns 8 i + 2 (lane % 4) (+1)
  const int lane = tid & 31, fr = 16 * warp + (lane >> 2), fc = 2 * (lane & 3);

  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    int t = tile;
    const int tw = t % tiles_w; t /= tiles_w;
    const int th = t % tiles_h;
    const int n = t / tiles_h;
    const int oy0 = th * CFT_TH, ox0 = tw * CFT_TW;
    const int iy0 = 2 * oy0 - 1, ix0 = 2 * ox0 - 1;  // SAME padding for k = 4, s = 2: one pixel before
    // ---- input patch (coalesced over the 3-channel pixels of a row), zero outside the image
    for (int i = tid; i < (int)CFT_PATCH_FLOATS; i += 128) {
      const int c = i % 3, px = (i / 3) % CFT_PW, py = i / (3 * CFT_PW);
      const int iy = iy0 + py, ix = ix0 + px;
      patch[i] = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? x[(((long long)n * H + iy) * W + ix) * 3 + c] : 0.f;
    }
    __syncthreads();
    // ---- this pixel's 48 taps -> row `tid` of A_hi / A_lo: tap k = (kh*4 + kw)*3 + c, 8 taps per 16-byte chunk
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int k = j * 8 + 2 * e + u;  // compile-time after unrolling
          if (k < 48) {
            const int kh = k / 12, kw = (k / 3) % 4, c = k % 3;
            v[u] = patch[((2 * ly + kh) * CFT_PW + (2 * lx + kw)) * 3 + c];
          } else {
            v[u] = 0.f;
          }
        }
        const __nv_bfloat162 h2 = __floats2bfloat162_rn(v[0], v[1]);
        const float2 hf = __bfloat1622float2(h2);
        hi[e] = *reinterpret_cast<const uint32_t*>(&h2);
        lo[e] = pack_bf16x2(v[0] - hf.x, v[1] - hf.y);
      }
      const uint32_t off = tid * 128 + (((j ^ (tid & 7)) & 7) << 4);
      st_shared_v4u(sAh + off, hi[0], hi[1], hi[2], hi[3]);
      st_shared_v4u(sAl + off, lo[0], lo[1], lo[2], lo[3]);
    }
    fence_proxy_async_smem();  // generic-proxy stores -> visible to wgmma (async proxy)
    __syncthreads();
    // ---- 64 x 64 output blocks: hi and lo products, then + bias, bf16, NHWC
    for (int mh = 0; mh < 2; ++mh) {
      const uint64_t dh = smem_desc_sw128(sAh + mh * 64 * 128, 0, 1024), dl = smem_desc_sw128(sAl + mh * 64 * 128, 0, 1024);
      for (int nb = 0; nb < Cout / 64; ++nb) {
        const uint64_t db = smem_desc_sw128(sB + nb * 64 * 128, 0, 1024);
        float d[32];
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_m64n64<0, 0>(d, dh + 2u * kk, db + 2u * kk, kk > 0);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_m64n64<0, 0>(d, dl + 2u * kk, db + 2u * kk, 1u);
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = mh * 64 + fr + 8 * h;
          const int oy = oy0 + r / CFT_TW, ox = ox0 + r % CFT_TW;
          if (oy >= Ho || ox >= Wo) continue;
          bf16* dst = y + (((long long)n * Ho + oy) * Wo + ox) * Cout + nb * 64 + fc;
          const float* bb = sbias + nb * 64 + fc;
#pragma unroll
          for (int i = 0; i < 8; ++i)
            *reinterpret_cast<uint32_t*>(dst + 8 * i) =
                pack_bf16x2(d[4 * i + 2 * h] + bb[8 * i], d[4 * i + 2 * h + 1] + bb[8 * i + 1]);
        }
      }
    }
    __syncthreads();  // A tiles and the patch are free for the next tile
  }
}

int conv_first_tc_launch(cudaStream_t stream, const float* x, const float* w, const float* bias, void* y_bf16, int N,
                         int H, int W, int Cout) {
  const int Ho = H / 2, Wo = W / 2;
  const int tiles = ((Wo + CFT_TW - 1) / CFT_TW) * ((Ho + CFT_TH - 1) / CFT_TH) * N;
  const size_t smem = 1024 + 2 * CFT_A_BYTES + (size_t)Cout * 128 + CFT_PATCH_FLOATS * 4 + (size_t)Cout * 4 + 64;
  static const cudaError_t attr_rc = cudaFuncSetAttribute(conv_first_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                          96 * 1024);  // once, thread-safe
  DB200_CUDA(attr_rc);
  // several CTAs per SM hide each other's gather / MMA / store phases (smem ~50 KB each)
  int grid = sm_count() * 4;
  if (grid > tiles) grid = tiles;
  conv_first_tc_kernel<<<grid, 128, smem, stream>>>(x, w, bias, reinterpret_cast<bf16*>(y_bf16), N, H, W, Cout);
  return check_launch("conv_first_tc_kernel");
}

}  // namespace db200
