// K11p — the DALL-E paper's discrete-VAE network: the 7x7 input convolution of the encoder (forward and weight
// gradient), 2x2 max-pool and 2x nearest-neighbour upsampling (forward and backward), and the residual blocks'
// post-gain / pre-activation pointwise step.  The blocks' 1x1 and 3x3 convolutions run on K11's kernels.
//
// Definition: oracle/vae_paper.py and DESIGN.md ("The DALL-E paper's dVAE network").  All element offsets are 64-bit:
// group-1 activations at 256^2 reach 2^31 elements at 128 images.
#include "common.cuh"
#include "ptx.cuh"

namespace db200 {

namespace {

template <typename T> __device__ __forceinline__ float ld(const T* p);
template <> __device__ __forceinline__ float ld<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ld<bf16>(const bf16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void st(T* p, float v);
template <> __device__ __forceinline__ void st<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void st<bf16>(bf16* p, float v) { *p = __float2bfloat16(v); }
template <typename T> __device__ __forceinline__ float rnd(float v);   // v as the activation type stores it
template <> __device__ __forceinline__ float rnd<float>(float v) { return v; }
template <> __device__ __forceinline__ float rnd<bf16>(float v) { return __bfloat162float(__float2bfloat16(v)); }

// ---------------------------------------------------------------------------------------------------------------
// 7x7 input conv, forward.  CTA: an 8 x 16 tile of output pixels of one image and 64 output channels; one pixel per
// thread with 64 f32 accumulators.  The (8+6) x (16+6) x C input patch and the 49 C x 64 kernel slice are staged in
// shared memory; weights are read as broadcast float4.  The image is read as f32 (the cast is fused).
// ---------------------------------------------------------------------------------------------------------------
constexpr int C7_TH = 8, C7_TW = 16, C7_PH = C7_TH + 6, C7_PW = C7_TW + 6;

template <typename TO>
__global__ void __launch_bounds__(128)
conv7_in_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                    TO* __restrict__ y, int H, int W, int C, int Cout) {
  extern __shared__ float c7_smem[];
  float* sw = c7_smem;                       // [49 C][64]
  float* sx = c7_smem + 49 * C * 64;         // [PH][PW][C]
  const int tiles_w = (W + C7_TW - 1) / C7_TW, tiles_h = (H + C7_TH - 1) / C7_TH;
  long long t = blockIdx.x;
  const int tw = (int)(t % tiles_w); t /= tiles_w;
  const int th = (int)(t % tiles_h); t /= tiles_h;
  const long long n = t;
  const int c0 = blockIdx.y * 64;
  const int oy0 = th * C7_TH, ox0 = tw * C7_TW;
  for (int i = threadIdx.x; i < 49 * C * 64; i += 128) {
    const int k = i >> 6, j = i & 63;
    sw[i] = (c0 + j < Cout) ? w[(long long)k * Cout + c0 + j] : 0.f;
  }
  for (int i = threadIdx.x; i < C7_PH * C7_PW * C; i += 128) {
    const int c = i % C, px = (i / C) % C7_PW, py = i / (C * C7_PW);
    const int iy = oy0 - 3 + py, ix = ox0 - 3 + px;
    sx[i] = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? x[((n * H + iy) * W + ix) * C + c] : 0.f;
  }
  __syncthreads();
  const int ly = threadIdx.x / C7_TW, lx = threadIdx.x % C7_TW;
  float acc[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = (bias && c0 + j < Cout) ? bias[c0 + j] : 0.f;
  for (int kh = 0; kh < 7; ++kh)
#pragma unroll
    for (int kw = 0; kw < 7; ++kw)
      for (int c = 0; c < C; ++c) {
        const float xv = sx[((ly + kh) * C7_PW + (lx + kw)) * C + c];
        const float4* wr = reinterpret_cast<const float4*>(sw + ((kh * 7 + kw) * C + c) * 64);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float4 wv = wr[j];
          acc[j * 4 + 0] = fmaf(xv, wv.x, acc[j * 4 + 0]);
          acc[j * 4 + 1] = fmaf(xv, wv.y, acc[j * 4 + 1]);
          acc[j * 4 + 2] = fmaf(xv, wv.z, acc[j * 4 + 2]);
          acc[j * 4 + 3] = fmaf(xv, wv.w, acc[j * 4 + 3]);
        }
      }
  const int oy = oy0 + ly, ox = ox0 + lx;
  if (oy >= H || ox >= W) return;
  TO* dst = y + ((n * H + oy) * W + ox) * Cout + c0;
#pragma unroll
  for (int j = 0; j < 64; j += 8) {
    if (c0 + j >= Cout) break;
    if constexpr (sizeof(TO) == 2) {
      uint4 q;
      q.x = pack_bf16x2(acc[j], acc[j + 1]); q.y = pack_bf16x2(acc[j + 2], acc[j + 3]);
      q.z = pack_bf16x2(acc[j + 4], acc[j + 5]); q.w = pack_bf16x2(acc[j + 6], acc[j + 7]);
      *reinterpret_cast<uint4*>(dst + j) = q;
    } else {
      *reinterpret_cast<float4*>(dst + j) = make_float4(acc[j], acc[j + 1], acc[j + 2], acc[j + 3]);
      *reinterpret_cast<float4*>(dst + j + 4) = make_float4(acc[j + 4], acc[j + 5], acc[j + 6], acc[j + 7]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// 7x7 input conv, weight gradient.  CTA (64 output channels, pixel split, kernel row kh): thread (co = tid & 63, lane
// group tid >> 6) streams the split's pixels 4 apart (dy coalesced over co, the image values warp-broadcast) and keeps
// the 7 C accumulators of row kh (+ the bias on kh == 0).  The 4 lane groups are added in order through shared memory
// and the CTA stores its partial into the workspace row of its split; reduce_rows_add sums the splits in order.
// ---------------------------------------------------------------------------------------------------------------
template <typename TD>
__global__ void __launch_bounds__(256)
conv7_in_wgrad_kernel(const float* __restrict__ x, const TD* __restrict__ dy, float* __restrict__ ws_w,
                      float* __restrict__ ws_b, int H, int W, int C, int Cout, long long M, long long per) {
  __shared__ float red[4][64];
  const int c = threadIdx.x & 63, pl = threadIdx.x >> 6;
  const int co = blockIdx.x * 64 + c;
  const int split = blockIdx.y, kh = blockIdx.z;
  const bool ok = co < Cout;
  const long long mbeg = (long long)split * per, mend = mbeg + per < M ? mbeg + per : M;
  float acc[7][4], accb = 0.f;
#pragma unroll
  for (int i = 0; i < 7; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (long long m = mbeg + pl; m < mend; m += 4) {
    const int ox = (int)(m % W);
    const long long r = m / W;
    const int oy = (int)(r % H);
    const long long n = r / H;
    const float dv = ok ? ld<TD>(dy + m * Cout + co) : 0.f;
    accb += dv;
    const int iy = oy + kh - 3;
    if (iy < 0 || iy >= H) continue;
    const float* row = x + (n * H + iy) * W * C;
#pragma unroll
    for (int kw = 0; kw < 7; ++kw) {
      const int ix = ox + kw - 3;
      if (ix < 0 || ix >= W) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < C) acc[kw][j] = fmaf(row[(long long)ix * C + j], dv, acc[kw][j]);
    }
  }
  const long long row_w = 49ll * C * Cout;
#pragma unroll
  for (int kw = 0; kw < 7; ++kw)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j >= C) break;
      red[pl][c] = acc[kw][j];
      __syncthreads();
      if (pl == 0 && ok)
        ws_w[split * row_w + ((long long)(kh * 7 + kw) * C + j) * Cout + co] =
            ((red[0][c] + red[1][c]) + red[2][c]) + red[3][c];
      __syncthreads();
    }
  if (kh == 0 && ws_b) {
    red[pl][c] = accb;
    __syncthreads();
    if (pl == 0 && ok) ws_b[(long long)split * Cout + co] = ((red[0][c] + red[1][c]) + red[2][c]) + red[3][c];
  }
}

int conv7_wgrad_splits(long long M, int Cout) {
  const int cblocks = (Cout + 63) / 64;
  long long splits = ((long long)sm_count() * 8 + cblocks * 7 - 1) / (cblocks * 7);
  const long long max_splits = (M + 255) / 256;   // >= 64 pixels per lane group
  if (splits > max_splits) splits = max_splits;
  return splits < 1 ? 1 : (int)splits;
}

// ---------------------------------------------------------------------------------------------------------------
// pointwise kernels: one element (max-pool / upsample: one low-resolution element) per thread, grid-stride
// ---------------------------------------------------------------------------------------------------------------
__host__ __device__ inline unsigned grid_for(long long n) {
  const long long b = (n + 255) / 256;
  return (unsigned)(b < 65535ll * 32 ? b : 65535ll * 32);
}

template <typename T>
__global__ void __launch_bounds__(256)
maxpool_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int H, int W, int C, long long n_out) {
  const int Wo = W / 2, Ho = H / 2;
  for (long long o = blockIdx.x * 256ll + threadIdx.x; o < n_out; o += (long long)gridDim.x * 256) {
    const int c = (int)(o % C);
    long long r = o / C;
    const int ox = (int)(r % Wo); r /= Wo;
    const int oy = (int)(r % Ho);
    const long long n = r / Ho;
    const long long i00 = ((n * H + 2 * oy) * W + 2 * ox) * C + c, i10 = i00 + (long long)W * C;
    float best = ld<T>(x + i00);
    const float v01 = ld<T>(x + i00 + C), v10 = ld<T>(x + i10), v11 = ld<T>(x + i10 + C);
    if (v01 > best) best = v01;
    if (v10 > best) best = v10;
    if (v11 > best) best = v11;
    st<T>(y + o, best);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
maxpool_bwd_kernel(const T* __restrict__ x, const T* __restrict__ dy, T* __restrict__ dx, int H, int W, int C,
                   long long n_out) {
  const int Wo = W / 2, Ho = H / 2;
  for (long long o = blockIdx.x * 256ll + threadIdx.x; o < n_out; o += (long long)gridDim.x * 256) {
    const int c = (int)(o % C);
    long long r = o / C;
    const int ox = (int)(r % Wo); r /= Wo;
    const int oy = (int)(r % Ho);
    const long long n = r / Ho;
    const long long i00 = ((n * H + 2 * oy) * W + 2 * ox) * C + c, row = (long long)W * C;
    const long long id[4] = {i00, i00 + C, i00 + row, i00 + row + C};
    float best = ld<T>(x + id[0]);
    int k = 0;
#pragma unroll
    for (int j = 1; j < 4; ++j) {
      const float v = ld<T>(x + id[j]);
      if (v > best) { best = v; k = j; }   // strictly greater: the first maximum keeps the gradient
    }
    const float g = ld<T>(dy + o);
#pragma unroll
    for (int j = 0; j < 4; ++j) st<T>(dx + id[j], j == k ? g : 0.f);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
upsample_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int H, int W, int C, long long n_in) {
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n_in; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int ix = (int)(r % W); r /= W;
    const int iy = (int)(r % H);
    const long long n = r / H;
    const T v = x[i];
    const long long o = ((n * 2 * H + 2 * iy) * 2 * W + 2 * ix) * C + c, row = 2ll * W * C;
    y[o] = v; y[o + C] = v; y[o + row] = v; y[o + row + C] = v;
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
upsample_bwd_kernel(const T* __restrict__ dy, T* __restrict__ dx, int H, int W, int C, long long n_in) {
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n_in; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int ix = (int)(r % W); r /= W;
    const int iy = (int)(r % H);
    const long long n = r / H;
    const long long o = ((n * 2 * H + 2 * iy) * 2 * W + 2 * ix) * C + c, row = 2ll * W * C;
    const float s = ((ld<T>(dy + o) + ld<T>(dy + o + C)) + ld<T>(dy + o + row)) + ld<T>(dy + o + row + C);
    st<T>(dx + i, s);
  }
}

// y may alias r or id: each element is read before it is written, by the same thread
template <typename T>
__global__ void __launch_bounds__(256)
residual_gain_kernel(const T* id, const T* r, const T* __restrict__ mask, float gain, T* y, T* relu_y, long long n) {
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    float v = id ? fmaf(gain, ld<T>(r + i), ld<T>(id + i)) : gain * ld<T>(r + i);
    if (mask && !(ld<T>(mask + i) > 0.f)) v = 0.f;
    v = rnd<T>(v);
    if (y) st<T>(y + i, v);
    if (relu_y) st<T>(relu_y + i, fmaxf(v, 0.f));
  }
}

int pool_check(const void* a, const void* b, const void* c, int N, int H, int W, int C, const char* who) {
  DB200_REQUIRE(a && b && c, DB200_E_INVALID, "%s: NULL pointer", who);
  DB200_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0, DB200_E_INVALID, "%s: non-positive dimension", who);
  return DB200_OK;
}

}  // namespace
}  // namespace db200

using namespace db200;

extern "C" int db200_conv7x7_in_fwd(db200_stream_t stream_, const float* x, const float* w, const float* bias, void* y,
                                    int N, int H, int W, int C, int Cout, int act_f32) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(x && w && y && N > 0 && H > 0 && W > 0 && Cout > 0, DB200_E_INVALID, "conv7x7_in_fwd: bad arguments");
  DB200_REQUIRE(C >= 1 && C <= 4 && Cout % 8 == 0, DB200_E_UNSUPPORTED,
                "conv7x7_in_fwd: needs 1 <= C <= 4 and Cout % 8 == 0 (C %d, Cout %d)", C, Cout);
  DB200_REQUIRE(aligned16(y), DB200_E_ALIGN, "conv7x7_in_fwd: unaligned output");
  const long long tiles = (long long)((W + C7_TW - 1) / C7_TW) * ((H + C7_TH - 1) / C7_TH) * N;
  DB200_REQUIRE(tiles < (1ll << 31), DB200_E_UNSUPPORTED, "conv7x7_in_fwd: too many tiles");
  const size_t smem = (size_t)(49 * C * 64 + C7_PH * C7_PW * C) * sizeof(float);
  if (smem > 48 * 1024) {
    static const cudaError_t a0 =
        cudaFuncSetAttribute(conv7_in_fwd_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    static const cudaError_t a1 =
        cudaFuncSetAttribute(conv7_in_fwd_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    DB200_CUDA(a0);
    DB200_CUDA(a1);
  }
  dim3 grid((unsigned)tiles, (Cout + 63) / 64);
  if (act_f32)
    conv7_in_fwd_kernel<float><<<grid, 128, smem, stream>>>(x, w, bias, reinterpret_cast<float*>(y), H, W, C, Cout);
  else
    conv7_in_fwd_kernel<bf16><<<grid, 128, smem, stream>>>(x, w, bias, reinterpret_cast<bf16*>(y), H, W, C, Cout);
  return check_launch("conv7_in_fwd_kernel");
}

extern "C" int64_t db200_conv7x7_in_wgrad_workspace_bytes(int N, int H, int W, int C, int Cout) {
  if (N <= 0 || H <= 0 || W <= 0 || C < 1 || C > 4 || Cout <= 0) return 0;
  const long long M = (long long)N * H * W;
  return (int64_t)conv7_wgrad_splits(M, Cout) * (49ll * C * Cout + Cout) * (int64_t)sizeof(float);
}

extern "C" int db200_conv7x7_in_wgrad(db200_stream_t stream_, const float* x, const void* dy, float* dw, float* dbias,
                                      int N, int H, int W, int C, int Cout, int act_f32, void* workspace,
                                      int64_t workspace_bytes) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(x && dy && dw && N > 0 && H > 0 && W > 0 && Cout > 0, DB200_E_INVALID,
                "conv7x7_in_wgrad: bad arguments");
  DB200_REQUIRE(C >= 1 && C <= 4, DB200_E_UNSUPPORTED, "conv7x7_in_wgrad: needs 1 <= C <= 4 (C %d)", C);
  const long long M = (long long)N * H * W;
  const int splits = conv7_wgrad_splits(M, Cout);
  const long long row_w = 49ll * C * Cout;
  DB200_REQUIRE(row_w < (1ll << 31) && (long long)splits * (row_w + Cout) < (1ll << 40), DB200_E_UNSUPPORTED,
                "conv7x7_in_wgrad: kernel too large");
  DB200_REQUIRE(workspace_ok(workspace, workspace_bytes, db200_conv7x7_in_wgrad_workspace_bytes(N, H, W, C, Cout)),
                DB200_E_INVALID, "conv7x7_in_wgrad: workspace too small or unaligned");
  float* ws_w = reinterpret_cast<float*>(workspace);
  float* ws_b = dbias ? ws_w + (long long)splits * row_w : nullptr;
  const long long per = (M + splits - 1) / splits;
  dim3 grid((Cout + 63) / 64, splits, 7);
  if (act_f32)
    conv7_in_wgrad_kernel<float><<<grid, 256, 0, stream>>>(x, reinterpret_cast<const float*>(dy), ws_w, ws_b, H, W, C,
                                                           Cout, M, per);
  else
    conv7_in_wgrad_kernel<bf16><<<grid, 256, 0, stream>>>(x, reinterpret_cast<const bf16*>(dy), ws_w, ws_b, H, W, C,
                                                          Cout, M, per);
  int rc = check_launch("conv7_in_wgrad_kernel");
  if (rc != DB200_OK) return rc;
  rc = reduce_rows_add(stream, ws_w, splits, (int)row_w, dw);
  if (rc != DB200_OK || !dbias) return rc;
  return reduce_rows_add(stream, ws_b, splits, Cout, dbias);
}

extern "C" int db200_maxpool2x2_fwd(db200_stream_t stream_, const void* x, void* y, int N, int H, int W, int C,
                                    int act_f32) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = pool_check(x, y, y, N, H, W, C, "maxpool2x2_fwd");
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(H % 2 == 0 && W % 2 == 0, DB200_E_UNSUPPORTED, "maxpool2x2_fwd: needs even H, W (%d x %d)", H, W);
  const long long n_out = (long long)N * (H / 2) * (W / 2) * C;
  if (act_f32)
    maxpool_fwd_kernel<float><<<grid_for(n_out), 256, 0, stream>>>((const float*)x, (float*)y, H, W, C, n_out);
  else
    maxpool_fwd_kernel<bf16><<<grid_for(n_out), 256, 0, stream>>>((const bf16*)x, (bf16*)y, H, W, C, n_out);
  return check_launch("maxpool_fwd_kernel");
}

extern "C" int db200_maxpool2x2_bwd(db200_stream_t stream_, const void* x, const void* dy, void* dx, int N, int H,
                                    int W, int C, int act_f32) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = pool_check(x, dy, dx, N, H, W, C, "maxpool2x2_bwd");
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(H % 2 == 0 && W % 2 == 0, DB200_E_UNSUPPORTED, "maxpool2x2_bwd: needs even H, W (%d x %d)", H, W);
  const long long n_out = (long long)N * (H / 2) * (W / 2) * C;
  if (act_f32)
    maxpool_bwd_kernel<float><<<grid_for(n_out), 256, 0, stream>>>((const float*)x, (const float*)dy, (float*)dx, H,
                                                                    W, C, n_out);
  else
    maxpool_bwd_kernel<bf16><<<grid_for(n_out), 256, 0, stream>>>((const bf16*)x, (const bf16*)dy, (bf16*)dx, H, W,
                                                                   C, n_out);
  return check_launch("maxpool_bwd_kernel");
}

extern "C" int db200_upsample2x_fwd(db200_stream_t stream_, const void* x, void* y, int N, int H, int W, int C,
                                    int act_f32) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = pool_check(x, y, y, N, H, W, C, "upsample2x_fwd");
  if (rc != DB200_OK) return rc;
  const long long n_in = (long long)N * H * W * C;
  if (act_f32)
    upsample_fwd_kernel<float><<<grid_for(n_in), 256, 0, stream>>>((const float*)x, (float*)y, H, W, C, n_in);
  else
    upsample_fwd_kernel<bf16><<<grid_for(n_in), 256, 0, stream>>>((const bf16*)x, (bf16*)y, H, W, C, n_in);
  return check_launch("upsample_fwd_kernel");
}

extern "C" int db200_upsample2x_bwd(db200_stream_t stream_, const void* dy, void* dx, int N, int H, int W, int C,
                                    int act_f32) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = pool_check(dy, dx, dx, N, H, W, C, "upsample2x_bwd");
  if (rc != DB200_OK) return rc;
  const long long n_in = (long long)N * H * W * C;
  if (act_f32)
    upsample_bwd_kernel<float><<<grid_for(n_in), 256, 0, stream>>>((const float*)dy, (float*)dx, H, W, C, n_in);
  else
    upsample_bwd_kernel<bf16><<<grid_for(n_in), 256, 0, stream>>>((const bf16*)dy, (bf16*)dx, H, W, C, n_in);
  return check_launch("upsample_bwd_kernel");
}

extern "C" int db200_residual_gain(db200_stream_t stream_, const void* id, const void* r, const void* mask,
                                   float gain, void* y, void* relu_y, int64_t n, int act_f32) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(r && (y || relu_y) && n > 0, DB200_E_INVALID, "residual_gain: bad arguments");
  DB200_REQUIRE(std::isfinite(gain), DB200_E_INVALID, "residual_gain: gain must be finite");
  if (act_f32)
    residual_gain_kernel<float><<<grid_for(n), 256, 0, stream>>>((const float*)id, (const float*)r,
                                                                 (const float*)mask, gain, (float*)y, (float*)relu_y,
                                                                 (long long)n);
  else
    residual_gain_kernel<bf16><<<grid_for(n), 256, 0, stream>>>((const bf16*)id, (const bf16*)r, (const bf16*)mask,
                                                                gain, (bf16*)y, (bf16*)relu_y, (long long)n);
  return check_launch("residual_gain_kernel");
}
