// K11 — discrete-VAE convolutions as im2col-free, shared-memory-staged direct convolutions (CUDA cores, fp32
// accumulate).  One generic "gather-GEMM" kernel covers conv / conv-transpose forward and both dgrads, one generic
// "outer-product" kernel covers both wgrads; the host describes each case with a tap list.
//
//   gather-GEMM:   y[pix, n] = epi( sum_taps sum_k  x[src(pix, tap), k] * w[tap][k][n] )
//                  64 pixels x 64 channels per CTA, K staged through smem in chunks of 16, 4x4 outputs per thread.
//   outer-product: dw[tap][a][b] += sum_pix p[srcP(pix,tap), a] * q[srcQ(pix,tap), b]   (split over pixels, red.add)
//
// Reference: tf.layers.conv2d / conv2d_transpose call sites src/vae_tf/models.py:95-109, 139-155 (NHWC, HWIO,
// padding SAME); codebook matmuls src/vae_tf/models.py:118,127 reuse the same kernels with a 1x1 geometry.
#include "common.cuh"
#include "ptx.cuh"
#include "conv_params.cuh"

namespace db200 {

template <typename T> __device__ __forceinline__ float ldf(const T* p);
template <> __device__ __forceinline__ float ldf<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ldf<bf16>(const bf16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void stf(T* p, float v);
template <> __device__ __forceinline__ void stf<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void stf<bf16>(bf16* p, float v) { *p = __float2bfloat16(v); }

template <typename T>
__global__ void __launch_bounds__(256)
conv_gemm_kernel(const ConvGemmParams p) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long long M = (long long)p.NB * p.OH * p.OW;
  const long long m0 = (long long)blockIdx.x * 64;
  const int n0 = blockIdx.y * 64;
  const T* x = reinterpret_cast<const T*>(p.x);

  // A loader: this thread always stages pixel (tid >> 2), channels ((tid & 3) * 4 .. +3) of the current K chunk
  const int a_pix = tid >> 2, a_k = (tid & 3) * 4;
  const long long am = m0 + a_pix;
  int a_n = 0, a_oy = 0, a_ox = 0;
  const bool a_ok = am < M;
  if (a_ok) {
    a_ox = (int)(am % p.OW);
    a_oy = (int)((am / p.OW) % p.OH);
    a_n = (int)(am / ((long long)p.OW * p.OH));
  }
  const bool n_contig = (p.w_n_stride == 1);

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int t = 0; t < p.ntaps; ++t) {
    const int iy = a_oy * p.in_stride + p.taps[t].dy, ix = a_ox * p.in_stride + p.taps[t].dx;
    const bool src_ok = a_ok && iy >= 0 && iy < p.in_H && ix >= 0 && ix < p.in_W;
    const T* src = x + (((long long)a_n * p.in_H + iy) * p.in_W + ix) * p.K;
    const float* wt = p.w + p.taps[t].w_off;
    for (int k0 = 0; k0 < p.K; k0 += 16) {
      // ---- stage A (zero-filled outside the image / beyond K)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = k0 + a_k + j;
        As[a_k + j][a_pix] = (src_ok && k < p.K) ? ldf<T>(src + k) : 0.f;
      }
      // ---- stage B
      if (n_contig) {
        const int bk = tid >> 4, bn = (tid & 15) * 4;
        const int k = k0 + bk;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int n = n0 + bn + j;
          Bs[bk][bn + j] = (k < p.K && n < p.Nn) ? wt[(long long)k * p.w_k_stride + n] : 0.f;
        }
      } else {
        const int bn = tid >> 2, bk = (tid & 3) * 4;
        const int n = n0 + bn;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int k = k0 + bk + j;
          Bs[bk + j][bn] = (k < p.K && n < p.Nn) ? wt[(long long)k * p.w_k_stride + (long long)n * p.w_n_stride] : 0.f;
        }
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
  // ---- epilogue
  T* y = reinterpret_cast<T*>(p.y);
  const T* res = reinterpret_cast<const T*>(p.residual);
  const T* msk = reinterpret_cast<const T*>(p.mask);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const int ox = (int)(m % p.OW);
    const int oy = (int)((m / p.OW) % p.OH);
    const int n = (int)(m / ((long long)p.OW * p.OH));
    const long long o =
        (((long long)n * p.out_H + (oy * p.out_stride + p.oa)) * p.out_W + (ox * p.out_stride + p.ob)) * p.Nn;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = n0 + tx * 4 + j;
      if (c >= p.Nn) continue;
      float v = acc[i][j];
      if (p.bias) v += p.bias[c];
      if (p.relu) v = fmaxf(v, 0.f);
      if (msk) v = ldf<T>(msk + o + c) > 0.f ? v : 0.f;
      if (res) v += ldf<T>(res + o + c);
      stf<T>(y + o + c, v);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
conv_wgrad_kernel(const ConvWgradParams p) {
  __shared__ float Ps[16][64 + 4];
  __shared__ float Qs[16][64 + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int a0 = blockIdx.x * 64, b0 = blockIdx.y * 64;
  const int t = blockIdx.z % p.ntaps, split = blockIdx.z / p.ntaps;
  const long long M = (long long)p.NB * p.OH * p.OW;
  const long long per = ((M + p.splits - 1) / p.splits + 15) / 16 * 16;
  const long long mbeg = split * per, mend = (mbeg + per < M) ? mbeg + per : M;
  const T* P = reinterpret_cast<const T*>(p.P);
  const T* Q = reinterpret_cast<const T*>(p.Q);
  const WgradTap tap = p.taps[t];
  const int l_pix = tid >> 4, l_c = (tid & 15) * 4;  // loader: pixel l_pix of the chunk, channels l_c..l_c+3

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (long long mm = mbeg; mm < mend; mm += 16) {
    const long long m = mm + l_pix;
    bool pok = false, qok = false;
    const T *psrc = P, *qsrc = Q;
    if (m < mend) {
      const int ox = (int)(m % p.OW);
      const int oy = (int)((m / p.OW) % p.OH);
      const int n = (int)(m / ((long long)p.OW * p.OH));
      const int py = oy * p.p_stride + tap.pdy, px = ox * p.p_stride + tap.pdx;
      const int qy = oy * p.q_stride + tap.qdy, qx = ox * p.q_stride + tap.qdx;
      pok = py >= 0 && py < p.pH && px >= 0 && px < p.pW;
      qok = qy >= 0 && qy < p.qH && qx >= 0 && qx < p.qW;
      psrc = P + (((long long)n * p.pH + py) * p.pW + px) * p.pC;
      qsrc = Q + (((long long)n * p.qH + qy) * p.qW + qx) * p.qC;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int a = a0 + l_c + j, b = b0 + l_c + j;
      Ps[l_pix][l_c + j] = (pok && a < p.pC) ? ldf<T>(psrc + a) : 0.f;
      Qs[l_pix][l_c + j] = (qok && b < p.qC) ? ldf<T>(qsrc + b) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&Ps[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Qs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* dw = p.dw + tap.w_off;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int a = a0 + ty * 4 + i;
    if (a >= p.pC) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int b = b0 + tx * 4 + j;
      if (b >= p.qC) continue;
      atomicAdd(dw + (long long)a * p.a_stride + (long long)b * p.b_stride, acc[i][j]);
    }
  }
}

// column sums of a [rows][C] activation matrix (bias gradients), T = float | bf16
template <typename T>
__global__ void __launch_bounds__(256) colsum_act_kernel(const T* __restrict__ x, long long rows, int C,
                                                          float* __restrict__ out) {
  // block: 32 columns x 8 row-lanes
  __shared__ float red[8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  float acc = 0.f;
  if (c < C)
    for (long long r = (long long)blockIdx.y * 8 + ry; r < rows; r += (long long)gridDim.y * 8)
      acc += ldf<T>(x + r * C + c);
  red[ry][cx] = acc;
  __syncthreads();
  if (ry == 0 && c < C) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i][cx];
    atomicAdd(out + c, s);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// First encoder layer: 4x4 stride-2 SAME convolution of the fp32 image (Cin = 3) -> bf16 activations.
// K = 48 is far too small for the tensor pipe and the generic kernel wastes 5/6 of its 16-wide K chunks on padding,
// so this layer gets its own kernel: one output pixel per thread, a (2*8+2) x (2*16+2) x 3 input patch and the whole
// 4x4x3xCout kernel staged in shared memory, weights read as broadcast float4, 64 fp32 accumulators per thread,
// each thread stores its pixel's 64 channels as one contiguous 128-byte line.  Also absorbs the fp32 -> bf16 cast of
// the image.   Reference: the first conv_downsample of src/vae_tf/models.py:95.
// ---------------------------------------------------------------------------------------------------------------
constexpr int CF_TH = 8, CF_TW = 16;  // output tile per CTA (128 threads)
__global__ void __launch_bounds__(128)
conv_first_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                  bf16* __restrict__ y, int NB, int H, int W, int Cout) {
  extern __shared__ float cf_smem[];
  float* sw = cf_smem;                          // [48][Cout]
  float* sx = cf_smem + 48 * Cout;              // [(2*TH+2)][(2*TW+2)][3]
  constexpr int PH = 2 * CF_TH + 2, PW = 2 * CF_TW + 2;
  const int Ho = H / 2, Wo = W / 2;
  const int tiles_w = (Wo + CF_TW - 1) / CF_TW, tiles_h = (Ho + CF_TH - 1) / CF_TH;
  int t = blockIdx.x;
  const int tw = t % tiles_w; t /= tiles_w;
  const int th = t % tiles_h; t /= tiles_h;
  const int n = t;
  const int oy0 = th * CF_TH, ox0 = tw * CF_TW;
  for (int i = threadIdx.x; i < 48 * Cout; i += 128) sw[i] = w[i];
  const int iy0 = 2 * oy0 - 1, ix0 = 2 * ox0 - 1;  // SAME padding for k=4, s=2: one pixel before
  for (int i = threadIdx.x; i < PH * PW * 3; i += 128) {
    const int c = i % 3, px = (i / 3) % PW, py = i / (3 * PW);
    const int iy = iy0 + py, ix = ix0 + px;
    sx[i] = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? x[(((long long)n * H + iy) * W + ix) * 3 + c] : 0.f;
  }
  __syncthreads();
  const int ly = threadIdx.x / CF_TW, lx = threadIdx.x % CF_TW;
  const int oy = oy0 + ly, ox = ox0 + lx;
  float in[48];
#pragma unroll
  for (int kh = 0; kh < 4; ++kh)
#pragma unroll
    for (int kw = 0; kw < 4; ++kw)
#pragma unroll
      for (int c = 0; c < 3; ++c) in[(kh * 4 + kw) * 3 + c] = sx[((2 * ly + kh) * PW + (2 * lx + kw)) * 3 + c];
  for (int c0 = 0; c0 < Cout; c0 += 64) {
    float acc[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = bias ? bias[c0 + j] : 0.f;
#pragma unroll
    for (int k = 0; k < 48; ++k) {
      const float xv = in[k];
      const float4* wr = reinterpret_cast<const float4*>(sw + k * Cout + c0);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float4 wv = wr[j];  // same address for every thread: smem broadcast
        acc[j * 4 + 0] = fmaf(xv, wv.x, acc[j * 4 + 0]);
        acc[j * 4 + 1] = fmaf(xv, wv.y, acc[j * 4 + 1]);
        acc[j * 4 + 2] = fmaf(xv, wv.z, acc[j * 4 + 2]);
        acc[j * 4 + 3] = fmaf(xv, wv.w, acc[j * 4 + 3]);
      }
    }
    if (oy < Ho && ox < Wo) {
      bf16* dst = y + (((long long)n * Ho + oy) * Wo + ox) * Cout + c0;
#pragma unroll
      for (int j = 0; j < 64; j += 8) {
        uint4 q;
        q.x = pack_bf16x2(acc[j], acc[j + 1]); q.y = pack_bf16x2(acc[j + 2], acc[j + 3]);
        q.z = pack_bf16x2(acc[j + 4], acc[j + 5]); q.w = pack_bf16x2(acc[j + 6], acc[j + 7]);
        *reinterpret_cast<uint4*>(dst + j) = q;
      }
    }
  }
}

#ifdef DB200_DEV_KNOBS
static bool f32_fma_only() {   // development A/B switch: keep fp32 convolutions on the CUDA-core kernels
  static const bool v = [] { const char* e = getenv("DB200_CONV_F32_FMA"); return e && atoi(e) != 0; }();
  return v;
}
#else
static bool f32_fma_only() { return false; }
#endif

static int launch_gemm(cudaStream_t stream, const ConvGemmParams& p, bool act_f32) {
  const long long M = (long long)p.NB * p.OH * p.OW;
  if (act_f32 && !f32_fma_only() && conv_gemm_f32_tc_ok(p)) return conv_gemm_f32_tc_launch(stream, p);
  dim3 grid((unsigned)((M + 63) / 64), (unsigned)((p.Nn + 63) / 64));
  if (act_f32) conv_gemm_kernel<float><<<grid, 256, 0, stream>>>(p);
  else         conv_gemm_kernel<bf16><<<grid, 256, 0, stream>>>(p);
  return check_launch("conv_gemm_kernel");
}

// wgrad when one side has <= 4 channels (the RGB image on the first layer, the RGB output of the last 1x1 conv):
// the generic 64x64 outer-product tile would waste 94 % of its FMAs.  Here a CTA owns (tap, 64 channels of the wide
// side, pixel split); thread (c = tid & 63, lane-group = tid >> 6) streams pixels (coalesced over c) and keeps
// <= 4 accumulators; one smem reduction + <= 256 atomics per CTA.  HBM-bound.
struct SkinnyWgradParams {
  int NB, OH, OW;
  int wH, wW, wC, w_stride;   // wide tensor (64-channel slices)
  int nH, nW, nC, n_stride;   // narrow tensor (nC <= 4)
  int ntaps, splits;
  WgradTap taps[MAX_TAPS];    // pd* -> wide tensor offsets, qd* -> narrow tensor offsets
  long long wide_stride, narrow_stride;  // element strides of dw along the wide / narrow channel index
  const void* Wd;
  const void* Nr;
  float* dw;
};

template <typename T>
__global__ void __launch_bounds__(256)
conv_wgrad_skinny_kernel(const SkinnyWgradParams p) {
  // one pass over the pixels for ALL taps: the wide value is loaded once per pixel, the (<= 4-channel) narrow values
  // of each tap are warp-broadcast loads; MAX_TAPS x 4 accumulators per thread; 32-bit index arithmetic.
  __shared__ float red[4][64];
  const int c = threadIdx.x & 63, pl = threadIdx.x >> 6;
  const int c0 = blockIdx.x * 64;
  const int M = p.NB * p.OH * p.OW;
  const int per = (M + p.splits - 1) / p.splits;
  const int mbeg = blockIdx.y * per, mend = min(M, mbeg + per);
  const T* Wd = reinterpret_cast<const T*>(p.Wd);
  const T* Nr = reinterpret_cast<const T*>(p.Nr);
  float acc[MAX_TAPS][4];
#pragma unroll
  for (int t = 0; t < MAX_TAPS; ++t)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[t][j] = 0.f;
  const bool c_ok = c0 + c < p.wC;
  for (int m = mbeg + pl; m < mend; m += 4) {
    const int ox = m % p.OW;
    const int oy = (m / p.OW) % p.OH;
    const int n = m / (p.OW * p.OH);
    int last_wy = -0x7fffffff, last_wx = 0;
    float wv = 0.f;
#pragma unroll
    for (int t = 0; t < MAX_TAPS; ++t) {
      if (t >= p.ntaps) break;
      const int wy = oy * p.w_stride + p.taps[t].pdy, wx = ox * p.w_stride + p.taps[t].pdx;
      if (wy != last_wy || wx != last_wx) {
        const bool ok = c_ok && wy >= 0 && wy < p.wH && wx >= 0 && wx < p.wW;
        wv = ok ? ldf<T>(Wd + ((long long)(n * p.wH + wy) * p.wW + wx) * p.wC + c0 + c) : 0.f;
        last_wy = wy; last_wx = wx;
      }
      const int ny = oy * p.n_stride + p.taps[t].qdy, nx = ox * p.n_stride + p.taps[t].qdx;
      if (ny < 0 || ny >= p.nH || nx < 0 || nx >= p.nW) continue;
      const T* nr = Nr + ((long long)(n * p.nH + ny) * p.nW + nx) * p.nC;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < p.nC) acc[t][j] = fmaf(wv, ldf<T>(nr + j), acc[t][j]);
    }
  }
  for (int t = 0; t < p.ntaps; ++t)
    for (int j = 0; j < p.nC; ++j) {
      float v = 0.f;
#pragma unroll
      for (int tt = 0; tt < MAX_TAPS; ++tt)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
          if (tt == t && jj == j) v = acc[tt][jj];  // compile-time indexed registers
      red[pl][c] = v;
      __syncthreads();
      if (pl == 0 && c_ok)
        atomicAdd(p.dw + p.taps[t].w_off + (long long)(c0 + c) * p.wide_stride + (long long)j * p.narrow_stride,
                  red[0][c] + red[1][c] + red[2][c] + red[3][c]);
      __syncthreads();
    }
}

static int launch_wgrad(cudaStream_t stream, ConvWgradParams& p, bool act_f32) {
  if (p.pC <= 4 || p.qC <= 4) {
    SkinnyWgradParams q{};
    const bool p_narrow = p.pC <= 4 && !(p.qC <= 4 && p.qC < p.pC);
    q.NB = p.NB; q.OH = p.OH; q.OW = p.OW; q.ntaps = p.ntaps; q.dw = p.dw;
    for (int i = 0; i < p.ntaps; ++i) {
      q.taps[i] = p.taps[i];
      if (p_narrow) {  // wide = Q, narrow = P: swap the per-tap offsets so pd* always addresses the wide tensor
        q.taps[i].pdy = p.taps[i].qdy; q.taps[i].pdx = p.taps[i].qdx;
        q.taps[i].qdy = p.taps[i].pdy; q.taps[i].qdx = p.taps[i].pdx;
      }
    }
    if (p_narrow) {
      q.Wd = p.Q; q.wH = p.qH; q.wW = p.qW; q.wC = p.qC; q.w_stride = p.q_stride; q.wide_stride = p.b_stride;
      q.Nr = p.P; q.nH = p.pH; q.nW = p.pW; q.nC = p.pC; q.n_stride = p.p_stride; q.narrow_stride = p.a_stride;
    } else {
      q.Wd = p.P; q.wH = p.pH; q.wW = p.pW; q.wC = p.pC; q.w_stride = p.p_stride; q.wide_stride = p.a_stride;
      q.Nr = p.Q; q.nH = p.qH; q.nW = p.qW; q.nC = p.qC; q.n_stride = p.q_stride; q.narrow_stride = p.b_stride;
    }
    const long long M = (long long)p.NB * p.OH * p.OW;
    DB200_REQUIRE(M < (1ll << 31), DB200_E_UNSUPPORTED, "conv2d_wgrad: more than 2^31 pixels");
    const int cblocks = (q.wC + 63) / 64;
    int splits = (sm_count() * 8 + cblocks - 1) / cblocks;
    const long long max_splits = (M + 127) / 128;   // >= 32 pixels per lane group
    if (splits > max_splits) splits = (int)max_splits;
    if (splits < 1) splits = 1;
    q.splits = splits;
    dim3 grid(cblocks, splits);
    if (act_f32) conv_wgrad_skinny_kernel<float><<<grid, 256, 0, stream>>>(q);
    else         conv_wgrad_skinny_kernel<bf16><<<grid, 256, 0, stream>>>(q);
    return check_launch("conv_wgrad_skinny_kernel");
  }
  if (act_f32 && !f32_fma_only() && conv_wgrad_f32_tc_ok(p)) return conv_wgrad_f32_tc_launch(stream, p);
  const long long M = (long long)p.NB * p.OH * p.OW;
  const int tiles = ((p.pC + 63) / 64) * ((p.qC + 63) / 64) * p.ntaps;
  int splits = (sm_count() * 4 + tiles - 1) / tiles;
  const long long max_splits = (M + 255) / 256;  // at least 256 pixels per split
  if (splits > max_splits) splits = (int)max_splits;
  if (splits < 1) splits = 1;
  p.splits = splits;
  dim3 grid((p.pC + 63) / 64, (p.qC + 63) / 64, p.ntaps * splits);
  if (act_f32) conv_wgrad_kernel<float><<<grid, 256, 0, stream>>>(p);
  else         conv_wgrad_kernel<bf16><<<grid, 256, 0, stream>>>(p);
  return check_launch("conv_wgrad_kernel");
}

static int pad_before(int in, int out, int k, int s) {
  int total = (out - 1) * s + k - in;
  if (total < 0) total = 0;
  return total / 2;  // TF SAME: the odd pixel goes after
}

static int validate(const db200_conv_desc* c, const char* who) {
  DB200_REQUIRE(c != nullptr, DB200_E_INVALID, "%s: NULL descriptor", who);
  DB200_REQUIRE(c->N > 0 && c->H > 0 && c->W > 0 && c->Cin > 0 && c->Cout > 0 && c->Ho > 0 && c->Wo > 0,
                DB200_E_INVALID, "%s: non-positive dimension", who);
  DB200_REQUIRE(c->KH > 0 && c->KW > 0 && c->KH * c->KW <= MAX_TAPS, DB200_E_UNSUPPORTED,
                "%s: kernel %dx%d has more than %d taps", who, c->KH, c->KW, MAX_TAPS);
  DB200_REQUIRE(c->stride == 1 || c->stride == 2, DB200_E_UNSUPPORTED, "%s: stride %d not in {1,2}", who, c->stride);
  if (c->transposed) {
    DB200_REQUIRE(c->KH == 4 && c->KW == 4 && c->stride == 2 && c->Ho == 2 * c->H && c->Wo == 2 * c->W,
                  DB200_E_UNSUPPORTED, "%s: conv2d_transpose is implemented for k=4, s=2, SAME only", who);
  } else {
    DB200_REQUIRE(c->Ho == (c->H + c->stride - 1) / c->stride && c->Wo == (c->W + c->stride - 1) / c->stride,
                  DB200_E_INVALID, "%s: Ho/Wo do not match SAME padding", who);
  }
  return DB200_OK;
}

}  // namespace db200

using namespace db200;

// ---------------------------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------------------------
extern "C" int db200_conv2d_fwd(db200_stream_t stream_, const db200_conv_desc* c, const void* x, const float* w,
                                const float* bias, const void* residual, void* y) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = validate(c, "conv2d_fwd");
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(x && w && y, DB200_E_INVALID, "conv2d_fwd: NULL pointer");
  ConvGemmParams p{};
  p.x = x; p.w = w; p.bias = bias; p.residual = residual; p.mask = nullptr; p.y = y;
  p.relu = c->relu;
  p.K = c->Cin; p.Nn = c->Cout;
  p.in_H = c->H; p.in_W = c->W;
  p.out_H = c->Ho; p.out_W = c->Wo;
  if (!c->transposed) {
    // y[oy,ox] = sum_{kh,kw} x[oy*s + kh - pt, ox*s + kw - pl] * w[kh][kw][ci][co]
    const int pt = pad_before(c->H, c->Ho, c->KH, c->stride), pl = pad_before(c->W, c->Wo, c->KW, c->stride);
    p.NB = c->N; p.OH = c->Ho; p.OW = c->Wo;
    p.out_stride = 1; p.oa = 0; p.ob = 0; p.in_stride = c->stride;
    p.ntaps = c->KH * c->KW;
    for (int kh = 0; kh < c->KH; ++kh)
      for (int kw = 0; kw < c->KW; ++kw) {
        Tap& t = p.taps[kh * c->KW + kw];
        t.dy = kh - pt; t.dx = kw - pl;
        t.w_off = (long long)(kh * c->KW + kw) * c->Cin * c->Cout;
      }
    p.w_k_stride = c->Cout; p.w_n_stride = 1;
    return launch_gemm(stream, p, c->act_f32 != 0);
  }
  // conv2d_transpose(k=4,s=2,SAME), kernel [kh][kw][cout][cin]:  y[2i-1+kh, 2j-1+kw, co] += x[i,j,ci] * w[kh][kw][co][ci]
  // one launch per output parity (a,b); each uses the 2x2 taps that land on that parity.
  p.NB = c->N; p.OH = c->H; p.OW = c->W;
  p.out_stride = 2; p.in_stride = 1;
  p.w_k_stride = 1; p.w_n_stride = c->Cin;
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      p.oa = a; p.ob = b; p.ntaps = 0;
      for (int kh = 0; kh < 4; ++kh) {
        if (((a + 1 - kh) & 1) != 0) continue;
        for (int kw = 0; kw < 4; ++kw) {
          if (((b + 1 - kw) & 1) != 0) continue;
          Tap& t = p.taps[p.ntaps++];
          t.dy = (a + 1 - kh) / 2; t.dx = (b + 1 - kw) / 2;  // exact: the numerators are even
          t.w_off = (long long)(kh * 4 + kw) * c->Cout * c->Cin;
        }
      }
      rc = launch_gemm(stream, p, c->act_f32 != 0);
      if (rc != DB200_OK) return rc;
    }
  return DB200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// dgrad: dx = d(loss)/d(x) given dy; optional ReLU mask (dx *= x_mask > 0) and residual-gradient add
// ---------------------------------------------------------------------------------------------------------------
extern "C" int db200_conv2d_dgrad(db200_stream_t stream_, const db200_conv_desc* c, const void* dy, const float* w,
                                  const void* x_mask, const void* dres, void* dx) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = validate(c, "conv2d_dgrad");
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(dy && w && dx, DB200_E_INVALID, "conv2d_dgrad: NULL pointer");
  ConvGemmParams p{};
  p.x = dy; p.w = w; p.bias = nullptr; p.residual = dres; p.mask = x_mask; p.y = dx; p.relu = 0;
  p.K = c->Cout; p.Nn = c->Cin;
  p.in_H = c->Ho; p.in_W = c->Wo;   // the tensor being gathered is dy
  p.out_H = c->H; p.out_W = c->W;   // the tensor being produced is dx
  if (!c->transposed) {
    const int pt = pad_before(c->H, c->Ho, c->KH, c->stride), pl = pad_before(c->W, c->Wo, c->KW, c->stride);
    // forward: iy = oy*s + kh - pt  =>  dx[iy] += dy[oy] * w[kh][kw][ci][co]
    p.w_k_stride = 1; p.w_n_stride = c->Cout;  // B(k = co, n = ci) = w[tap][ci][co]
    if (c->stride == 1) {
      p.NB = c->N; p.OH = c->H; p.OW = c->W;
      p.out_stride = 1; p.oa = 0; p.ob = 0; p.in_stride = 1;
      p.ntaps = c->KH * c->KW;
      for (int kh = 0; kh < c->KH; ++kh)
        for (int kw = 0; kw < c->KW; ++kw) {
          Tap& t = p.taps[kh * c->KW + kw];
          t.dy = pt - kh; t.dx = pl - kw;  // oy = iy + pt - kh
          t.w_off = (long long)(kh * c->KW + kw) * c->Cin * c->Cout;
        }
      return launch_gemm(stream, p, c->act_f32 != 0);
    }
    // stride 2: input pixel iy = 2*i + a receives from taps with (a + pt - kh) even; oy = i + (a + pt - kh)/2
    DB200_REQUIRE(c->H % 2 == 0 && c->W % 2 == 0, DB200_E_UNSUPPORTED, "conv2d_dgrad: stride 2 needs even H, W");
    p.NB = c->N; p.OH = c->H / 2; p.OW = c->W / 2;
    p.out_stride = 2; p.in_stride = 1;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        p.oa = a; p.ob = b; p.ntaps = 0;
        for (int kh = 0; kh < c->KH; ++kh) {
          if (((a + pt - kh) & 1) != 0) continue;
          for (int kw = 0; kw < c->KW; ++kw) {
            if (((b + pl - kw) & 1) != 0) continue;
            DB200_REQUIRE(p.ntaps < MAX_TAPS, DB200_E_UNSUPPORTED, "conv2d_dgrad: too many taps");
            Tap& t = p.taps[p.ntaps++];
            // floor division of a possibly negative even number
            t.dy = (a + pt - kh) / 2; t.dx = (b + pl - kw) / 2;
            t.w_off = (long long)(kh * c->KW + kw) * c->Cin * c->Cout;
          }
        }
        rc = launch_gemm(stream, p, c->act_f32 != 0);
        if (rc != DB200_OK) return rc;
      }
    return DB200_OK;
  }
  // transposed forward y[2i-1+kh] += x[i]*w[kh][kw][co][ci]  =>  dx[i,ci] = sum dy[2i-1+kh, 2j-1+kw, co] * w[..][co][ci]
  p.NB = c->N; p.OH = c->H; p.OW = c->W;
  p.out_stride = 1; p.oa = 0; p.ob = 0; p.in_stride = 2;
  p.ntaps = 16;
  for (int kh = 0; kh < 4; ++kh)
    for (int kw = 0; kw < 4; ++kw) {
      Tap& t = p.taps[kh * 4 + kw];
      t.dy = kh - 1; t.dx = kw - 1;
      t.w_off = (long long)(kh * 4 + kw) * c->Cout * c->Cin;
    }
  p.w_k_stride = c->Cin; p.w_n_stride = 1;  // B(k = co, n = ci) = w[tap][co][ci]
  return launch_gemm(stream, p, c->act_f32 != 0);
}

// ---------------------------------------------------------------------------------------------------------------
// wgrad (+ bias grad): accumulate into dw / dbias
// ---------------------------------------------------------------------------------------------------------------
extern "C" int db200_conv2d_wgrad(db200_stream_t stream_, const db200_conv_desc* c, const void* x, const void* dy,
                                  float* dw, float* dbias) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = validate(c, "conv2d_wgrad");
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(x && dy && dw, DB200_E_INVALID, "conv2d_wgrad: NULL pointer");
  ConvWgradParams p{};
  p.P = x; p.Q = dy; p.dw = dw;
  p.pH = c->H; p.pW = c->W; p.pC = c->Cin;
  p.qH = c->Ho; p.qW = c->Wo; p.qC = c->Cout;
  p.ntaps = c->KH * c->KW;
  if (!c->transposed) {
    const int pt = pad_before(c->H, c->Ho, c->KH, c->stride), pl = pad_before(c->W, c->Wo, c->KW, c->stride);
    p.NB = c->N; p.OH = c->Ho; p.OW = c->Wo;  // contract over output pixels
    p.p_stride = c->stride; p.q_stride = 1;
    for (int kh = 0; kh < c->KH; ++kh)
      for (int kw = 0; kw < c->KW; ++kw) {
        WgradTap& t = p.taps[kh * c->KW + kw];
        t.pdy = kh - pt; t.pdx = kw - pl; t.qdy = 0; t.qdx = 0;
        t.w_off = (long long)(kh * c->KW + kw) * c->Cin * c->Cout;
      }
    p.a_stride = c->Cout; p.b_stride = 1;  // dw[tap][ci][co]
  } else {
    p.NB = c->N; p.OH = c->H; p.OW = c->W;  // contract over input (low-res) pixels
    p.p_stride = 1; p.q_stride = 2;
    for (int kh = 0; kh < 4; ++kh)
      for (int kw = 0; kw < 4; ++kw) {
        WgradTap& t = p.taps[kh * 4 + kw];
        t.pdy = 0; t.pdx = 0; t.qdy = kh - 1; t.qdx = kw - 1;
        t.w_off = (long long)(kh * 4 + kw) * c->Cout * c->Cin;
      }
    p.a_stride = 1; p.b_stride = c->Cin;  // dw[tap][co][ci]
  }
  rc = launch_wgrad(stream, p, c->act_f32 != 0);
  if (rc != DB200_OK) return rc;
  if (dbias) {
    const long long rows = (long long)c->N * c->Ho * c->Wo;
    dim3 grid((c->Cout + 31) / 32, (unsigned)((rows + 255) / 256 < 512 ? (rows + 255) / 256 : 512));
    if (c->act_f32) colsum_act_kernel<float><<<grid, 256, 0, stream>>>((const float*)dy, rows, c->Cout, dbias);
    else            colsum_act_kernel<bf16><<<grid, 256, 0, stream>>>((const bf16*)dy, rows, c->Cout, dbias);
    return check_launch("colsum_act_kernel");
  }
  return DB200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// small fp32 matmuls (codebook): the same kernels with a 1x1 geometry
// ---------------------------------------------------------------------------------------------------------------
extern "C" int db200_rowmatmul_f32(db200_stream_t stream_, const float* a, const float* b, float* out, int rows, int K,
                                   int N, int b_transposed, int accumulate) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(a && b && out && rows > 0 && K > 0 && N > 0, DB200_E_INVALID, "rowmatmul: bad arguments");
  ConvGemmParams p{};
  p.NB = rows; p.OH = 1; p.OW = 1; p.out_H = 1; p.out_W = 1; p.out_stride = 1; p.in_H = 1; p.in_W = 1; p.in_stride = 1;
  p.K = K; p.Nn = N; p.ntaps = 1;
  p.taps[0].dy = 0; p.taps[0].dx = 0; p.taps[0].w_off = 0;
  if (b_transposed) { p.w_k_stride = 1; p.w_n_stride = K; }  // b stored [N][K]
  else              { p.w_k_stride = N; p.w_n_stride = 1; }  // b stored [K][N]
  p.x = a; p.w = b; p.y = out;
  p.residual = accumulate ? out : nullptr;
  return launch_gemm(stream, p, true);
}

extern "C" int db200_rowmatmul_tn_f32(db200_stream_t stream_, const float* a, const float* b, float* out_accum,
                                      int rows, int M, int N) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(a && b && out_accum && rows > 0 && M > 0 && N > 0, DB200_E_INVALID, "rowmatmul_tn: bad arguments");
  ConvWgradParams p{};
  p.NB = rows; p.OH = 1; p.OW = 1;
  p.pH = 1; p.pW = 1; p.pC = M; p.p_stride = 1;
  p.qH = 1; p.qW = 1; p.qC = N; p.q_stride = 1;
  p.ntaps = 1;
  p.taps[0] = WgradTap{0, 0, 0, 0, 0};
  p.a_stride = N; p.b_stride = 1;
  p.P = a; p.Q = b; p.dw = out_accum;
  return launch_wgrad(stream, p, true);
}

namespace db200 {
int conv_first_tc_launch(cudaStream_t stream, const float* x, const float* w, const float* bias, void* y_bf16, int N,
                         int H, int W, int Cout);
}
// y (bf16 NHWC) = conv4x4/s2/SAME(x fp32 NHWC [N][H][W][3], w f32 [4][4][3][Cout]) + bias.   Cout % 64 == 0.
extern "C" int db200_conv2d_first_fwd(db200_stream_t stream_, const float* x, const float* w, const float* bias,
                                      void* y_bf16, int N, int H, int W, int Cout) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(x && w && y_bf16 && N > 0 && H > 0 && W > 0, DB200_E_INVALID, "conv2d_first_fwd: bad arguments");
  DB200_REQUIRE(H % 2 == 0 && W % 2 == 0 && Cout % 64 == 0 && Cout <= 256, DB200_E_UNSUPPORTED,
                "conv2d_first_fwd: needs even H, W and Cout in {64,128,192,256}");
  DB200_REQUIRE(aligned16(w) && aligned16(y_bf16), DB200_E_ALIGN, "conv2d_first_fwd: unaligned pointer");
  return conv_first_tc_launch(stream, x, w, bias, y_bf16, N, H, W, Cout);  // wgmma (conv_first_tc.cu)
}

// CUDA-core version of the first layer (fp32 FMA; kept for A/B measurements: FMA-bound at ~5x the tensor-core kernel)
extern "C" int db200_conv2d_first_fwd_fma(db200_stream_t stream_, const float* x, const float* w, const float* bias,
                                          void* y_bf16, int N, int H, int W, int Cout) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(x && w && y_bf16 && N > 0 && H % 2 == 0 && W % 2 == 0 && Cout % 64 == 0 && Cout <= 256,
                DB200_E_INVALID, "conv2d_first_fwd_fma: bad arguments");
  const int Ho = H / 2, Wo = W / 2;
  const int tiles = ((Wo + CF_TW - 1) / CF_TW) * ((Ho + CF_TH - 1) / CF_TH) * N;
  const size_t smem = (size_t)(48 * Cout + (2 * CF_TH + 2) * (2 * CF_TW + 2) * 3) * sizeof(float);
  if (smem > 48 * 1024) {
    static const cudaError_t attr_rc = cudaFuncSetAttribute(conv_first_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);  // once, thread-safe
    DB200_CUDA(attr_rc);
  }
  conv_first_kernel<<<tiles, 128, smem, stream>>>(x, w, bias, reinterpret_cast<bf16*>(y_bf16), N, H, W, Cout);
  return check_launch("conv_first_kernel");
}
