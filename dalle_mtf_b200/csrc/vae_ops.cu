// K13 — Gumbel-softmax (soft / hard straight-through), row argmax with the first-maximum tie rule, MSE loss.
// fp32 row kernels, one warp per row, warp-shuffle reductions; HBM-bound (the [rows][K] tensors are read/written once
// or twice).
//
// Reference: gumbel_softmax src/vae_tf/layers.py:4-21, mse_loss :24-25, tf.math.argmax src/model_fns.py:76.
#include "common.cuh"
#include "ptx.cuh"

namespace db200 {

// (value, index) max with "lowest index wins on ties" — tf.argmax / np.argmax semantics
__device__ __forceinline__ void argmax_combine(float& v, int& i, float ov, int oi) {
  if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
}
__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    argmax_combine(v, i, ov, oi);
  }
}

__global__ void __launch_bounds__(128)
gumbel_softmax_fwd_kernel(const float* __restrict__ logits, const float* __restrict__ u, float* __restrict__ y_soft,
                          float* __restrict__ y_out, int* __restrict__ idx_out, int rows, int K, float inv_tau,
                          int hard) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* lr = logits + (long long)row * K;
  const float* ur = u ? u + (long long)row * K : nullptr;
  float* ys = y_soft + (long long)row * K;
  // pass 1: z = (logit + g) / tau into y_soft, track max
  float mv = -INFINITY;
  for (int k = lane; k < K; k += 32) {
    float z = lr[k];
    if (ur) z += -logf(-logf(ur[k]));  // g = -log(-log(u)), src/vae_tf/layers.py:8-14
    z *= inv_tau;
    ys[k] = z;
    mv = fmaxf(mv, z);
  }
  mv = warp_max(mv);
  float s = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float e = expf(ys[k] - mv);
    ys[k] = e;
    s += e;
  }
  s = warp_sum(s);
  const float inv = 1.f / s;
  float* yo = y_out ? y_out + (long long)row * K : nullptr;
  // pass 3: y = e / s, and the first maximum of y itself (tf.argmax(y), layers.py:17): z's that differ by an ulp can
  // round to the same y, and then the lower index wins, so idx is not the argmax of z.  The search starts at index 0:
  // a row with a NaN or +inf logit has y = NaN everywhere, which no comparison accepts, and it then gets idx 0 (and
  // the hard one-hot stores stay inside the row) instead of an index past the end.
  float my = -INFINITY;
  int mi = 0;
  for (int k = lane; k < K; k += 32) {
    const float yk = ys[k] * inv;
    ys[k] = yk;
    if (yo) yo[k] = hard ? 0.f : yk;
    argmax_combine(my, mi, yk, k);
  }
  warp_argmax(my, mi);
  if (hard && yo) {
    __syncwarp();  // orders this lane's 1 after the zero another lane of the warp stored there
    if (lane == 0) yo[mi] = 1.f;  // hard: one_hot(argmax y) forward value (layers.py:17-19)
  }
  if (idx_out && lane == 0) idx_out[row] = mi;
}

__global__ void __launch_bounds__(128)
gumbel_softmax_bwd_kernel(const float* __restrict__ y_soft, const float* __restrict__ dy, float* __restrict__ dlogits,
                          int rows, int K, float inv_tau) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* y = y_soft + (long long)row * K;
  const float* d = dy + (long long)row * K;
  float dot = 0.f;
  for (int k = lane; k < K; k += 32) dot += y[k] * d[k];
  dot = warp_sum(dot);
  float* o = dlogits + (long long)row * K;
  for (int k = lane; k < K; k += 32) o[k] = y[k] * (d[k] - dot) * inv_tau;
}

__global__ void __launch_bounds__(128)
argmax_rows_kernel(const float* __restrict__ x, int* __restrict__ idx, int rows, int K) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + (long long)row * K;
  float mv = -INFINITY;
  int mi = 0;  // an all-NaN row yields 0, never an out-of-range token id
  for (int k = lane; k < K; k += 32) argmax_combine(mv, mi, xr[k], k);
  warp_argmax(mv, mi);
  if (lane == 0) idx[row] = mi;
}

__global__ void __launch_bounds__(256)
mse_kernel(const float* __restrict__ pred, const float* __restrict__ target, float* __restrict__ dpred,
           float* __restrict__ loss_accum, size_t n, float scale) {
  __shared__ float red[8];
  float acc = 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float d = pred[i] - target[i];
    acc += d * d;
    if (dpred) dpred[i] = 2.f * d * scale;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w];
    atomicAdd(loss_accum, s * scale);
  }
}

// tf.space_to_depth / tf.depth_to_space (NHWC, block size s) used by stack_factor > 1 (src/vae_tf/models.py:85-86,
// 155-161): deep[n, y, x, (dy*s + dx)*C + c] = flat[n, y*s + dy, x*s + dx, c].  One thread per element, coalesced on
// the deep side (the flat side is read / written in runs of C consecutive floats).
template <bool TO_DEPTH>
__global__ void __launch_bounds__(256)
space_depth_kernel(const float* __restrict__ in, float* __restrict__ out, long long n_elem, int Hd, int Wd, int C, int s) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // index on the deep side
  if (i >= n_elem) return;
  const int Cd = C * s * s;
  const int cd = (int)(i % Cd);
  long long t = i / Cd;
  const int x = (int)(t % Wd); t /= Wd;
  const int y = (int)(t % Hd);
  const long long n = t / Hd;
  const int c = cd % C, dx = (cd / C) % s, dy = cd / (C * s);
  const long long flat = ((n * (Hd * s) + (y * s + dy)) * (long long)(Wd * s) + (x * s + dx)) * C + c;
  if (TO_DEPTH) out[i] = in[flat];
  else          out[flat] = in[i];
}

}  // namespace db200

using namespace db200;

extern "C" int db200_space_to_depth_f32(db200_stream_t stream_, const float* in, float* out, int N, int H, int W, int C,
                                        int s, int inverse) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(in && out && N > 0 && s >= 1 && H % s == 0 && W % s == 0 && C > 0, DB200_E_INVALID,
                "space_to_depth: H, W must be multiples of the block size");
  const long long n = (long long)N * H * W * C;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  if (inverse) space_depth_kernel<false><<<blocks, 256, 0, stream>>>(in, out, n, H / s, W / s, C, s);
  else         space_depth_kernel<true><<<blocks, 256, 0, stream>>>(in, out, n, H / s, W / s, C, s);
  return check_launch("space_depth_kernel");
}

extern "C" int db200_gumbel_softmax_fwd(db200_stream_t stream_, const float* logits, const float* u, float* y_soft,
                                        float* y_out, int32_t* idx, int rows, int K, float tau, int hard) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(logits && y_soft && rows > 0 && K > 0 && tau > 0.f, DB200_E_INVALID,
                "gumbel_softmax_fwd: bad arguments");
  gumbel_softmax_fwd_kernel<<<(rows + 3) / 4, 128, 0, stream>>>(logits, u, y_soft, y_out, idx, rows, K, 1.f / tau,
                                                               hard);
  return check_launch("gumbel_softmax_fwd_kernel");
}

extern "C" int db200_gumbel_softmax_bwd(db200_stream_t stream_, const float* y_soft, const float* dy, float* dlogits,
                                        int rows, int K, float tau) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(y_soft && dy && dlogits && rows > 0 && K > 0 && tau > 0.f, DB200_E_INVALID,
                "gumbel_softmax_bwd: bad arguments");
  gumbel_softmax_bwd_kernel<<<(rows + 3) / 4, 128, 0, stream>>>(y_soft, dy, dlogits, rows, K, 1.f / tau);
  return check_launch("gumbel_softmax_bwd_kernel");
}

extern "C" int db200_argmax_rows_f32(db200_stream_t stream_, const float* x, int32_t* idx, int rows, int K) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(x && idx && rows > 0 && K > 0, DB200_E_INVALID, "argmax_rows: bad arguments");
  argmax_rows_kernel<<<(rows + 3) / 4, 128, 0, stream>>>(x, idx, rows, K);
  return check_launch("argmax_rows_kernel");
}

extern "C" int db200_mse_fwd_bwd(db200_stream_t stream_, const float* pred, const float* target, float* dpred,
                                 float* loss_accum, size_t n, float scale) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(pred && target && loss_accum && n > 0, DB200_E_INVALID, "mse: bad arguments");
  size_t blocks = (n + 255) / 256;
  if (blocks > (size_t)sm_count() * 8) blocks = (size_t)sm_count() * 8;
  mse_kernel<<<(int)blocks, 256, 0, stream>>>(pred, target, dpred, loss_accum, n, scale);
  return check_launch("mse_kernel");
}
