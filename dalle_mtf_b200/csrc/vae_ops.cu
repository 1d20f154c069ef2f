// K13 — Gumbel-softmax (soft / hard straight-through), row argmax with the first-maximum tie rule, MSE loss, the
// optional KL(q || Uniform(K)) term with its codebook-usage histogram, and the optional logit-Laplace reconstruction
// loss.
// fp32 row kernels, one warp per row, warp-shuffle reductions; HBM-bound (the [rows][K] tensors are read/written once
// or twice).
//
// Reference: gumbel_softmax src/vae_tf/layers.py:4-21, mse_loss :24-25, tf.math.argmax src/model_fns.py:76.
#include <cfloat>
#include <type_traits>

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

// KL = false: the straight-through Gumbel-softmax backward.  KL = true adds the gradient of c * KL(q || Uniform(K)),
// q = softmax(logits), in the same store: c q (l - lse - ent), with lse / ent of the row from vae_kl_stats_kernel.
template <bool KL>
__global__ void __launch_bounds__(128)
gumbel_softmax_bwd_kernel(const float* __restrict__ y_soft, const float* __restrict__ dy, float* __restrict__ dlogits,
                          int rows, int K, float inv_tau, const float* __restrict__ logits,
                          const float* __restrict__ lse, const float* __restrict__ ent, float c) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* y = y_soft + (long long)row * K;
  const float* d = dy + (long long)row * K;
  float dot = 0.f;
  for (int k = lane; k < K; k += 32) dot += y[k] * d[k];
  dot = warp_sum(dot);
  float* o = dlogits + (long long)row * K;
  if (KL) {
    const float* lr = logits + (long long)row * K;
    const float ls = lse[row], en = ent[row];
    for (int k = lane; k < K; k += 32) {
      const float z = lr[k] - ls;              // log q, formed from the logit: q = 0 still gives a finite factor
      o[k] = y[k] * (d[k] - dot) * inv_tau + c * expf(z) * (fmaxf(z, -FLT_MAX) - en);
    }
  } else {
    for (int k = lane; k < K; k += 32) o[k] = y[k] * (d[k] - dot) * inv_tau;
  }
}

// ---- KL(q || Uniform(K)) statistics of the encoder logits (the KL term of the DALL-E paper's ELB; the reference has
// none).  One warp per row, KL_WARPS rows in flight per CTA, CTAs striding over the rows.  A single pass keeps, per lane,
// the running maximum m, s = sum exp(l - m) and t = sum exp(l - m) (l - m), rescaled whenever m grows; then
//   lse = m + log s,   ent = sum q (l - lse) = t / s - log s,   KL_r = ent + log K = t / s - log(s / K)
// (the last form does not cancel log K against ent's -log K for near-uniform rows).  No log q is ever taken, so a q
// that underflows to 0 contributes exactly 0.
constexpr int KL_WARPS = 8;
constexpr int KL_SMEM_HIST_MAX_K = 12000;     // K * 4 bytes + red[] within the 48 KB a CTA gets without an opt-in

// (s, t) taken from maximum m to maximum mn >= m.  d is clamped so that an empty set (s = t = 0) stays 0, not 0 * -inf.
__device__ __forceinline__ void kl_rescale(float& s, float& t, float m, float mn) {
  const float a = expf(m - mn);
  t = a * fmaf(fmaxf(m - mn, -FLT_MAX), s, t);
  s = a * s;
}

// one logit l at index k into a lane's running (m, s, t), first maximum mi and NaN flag
__device__ __forceinline__ void kl_visit(float l, int k, float& m, float& s, float& t, int& mi, bool& nan) {
  nan |= l != l;
  if (l > m) {
    kl_rescale(s, t, m, l);
    s += 1.f;        // the new maximum itself: exp(0) = 1, (l - m) = 0
    m = l;
    mi = k;
  } else if (l != -INFINITY) {   // -inf has q = 0 and adds nothing; NaN falls through here and poisons s
    const float z = l - m;
    const float p = expf(z);
    s += p;
    t = fmaf(p, z, t);
  }
}

// VEC4 (K % 4 == 0, 16-byte aligned logits): a lane reads 4 consecutive logits per load, so a warp keeps four times the
// bytes in flight; a lane still visits its indices in increasing order, which keeps the first-maximum rule.
template <bool SMEM_HIST, bool VEC4>
__global__ void __launch_bounds__(KL_WARPS * 32)
vae_kl_stats_kernel(const float* __restrict__ logits, float* __restrict__ lse, float* __restrict__ ent,
                    int* __restrict__ hist, float* __restrict__ partials, int rows, int K, float Kf, float scale) {
  extern __shared__ int sh_hist[];
  __shared__ float red[KL_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int* h = hist;
  if (SMEM_HIST) {
    for (int k = threadIdx.x; k < K; k += blockDim.x) sh_hist[k] = 0;
    __syncthreads();
    h = sh_hist;
  }
  float kl_sum = 0.f;   // this warp's rows, in row order
  for (long long row = blockIdx.x * KL_WARPS + warp; row < rows; row += (long long)gridDim.x * KL_WARPS) {
    const float* lr = logits + (long long)row * K;
    float m = -INFINITY, s = 0.f, t = 0.f;
    int mi = 0;          // first index of the maximum (argmax_rows' rule); stays 0 for a row of -inf
    bool nan = false;
    if (VEC4) {
      const float4* lr4 = reinterpret_cast<const float4*>(lr);
#pragma unroll 2
      for (int j = lane; j < (K >> 2); j += 32) {
        const float4 v = lr4[j];
        kl_visit(v.x, 4 * j, m, s, t, mi, nan);
        kl_visit(v.y, 4 * j + 1, m, s, t, mi, nan);
        kl_visit(v.z, 4 * j + 2, m, s, t, mi, nan);
        kl_visit(v.w, 4 * j + 3, m, s, t, mi, nan);
      }
    } else {
#pragma unroll 4
      for (int k = lane; k < K; k += 32) kl_visit(lr[k], k, m, s, t, mi, nan);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, o);
      const float os = __shfl_xor_sync(0xffffffffu, s, o);
      const float ot = __shfl_xor_sync(0xffffffffu, t, o);
      const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
      const float mn = fmaxf(m, om);
      if (mn != -INFINITY) {   // else both halves hold only -inf logits (or none): s = t = 0 on both
        float s2 = os, t2 = ot;
        kl_rescale(s, t, m, mn);
        kl_rescale(s2, t2, om, mn);
        s += s2;
        t += t2;
      }
      if (om > m || (om == m && oi < mi)) mi = oi;
      m = mn;
    }
    nan = __any_sync(0xffffffffu, nan);
    const float ls = logf(s);
    const float ts = t / s;
    kl_sum += ts - logf(s / Kf);
    if (lane == 0) {
      lse[row] = m + ls;
      ent[row] = ts - ls;
      atomicAdd(&h[nan ? 0 : mi], 1);   // integer counts: exact in any order
    }
  }
  if (lane == 0) red[warp] = kl_sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < KL_WARPS; ++w) v += red[w];
    partials[blockIdx.x] = v * scale;   // per-CTA partial, summed in CTA order by the launcher
  }
  if (SMEM_HIST)
    for (int k = threadIdx.x; k < K; k += blockDim.x)
      if (sh_hist[k]) atomicAdd(&hist[k], sh_hist[k]);
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

// ---- logit-Laplace reconstruction loss (the DALL-E paper's dVAE likelihood; the reference has MSE only).  The decoder
// emits stats[p][0, Cp) = mu and stats[p][Cp, 2 Cp) = ln b per pixel p; the target x in [-1, 1] maps to
// y = clamp(eps + (1 - 2 eps)(x + 1) / 2, eps, 1 - eps) = clamp(0.4 x + 0.5, 0.1, 0.9), t = logit(y), and per subpixel
//   nll = ln 2 + ln b + ln y + ln(1 - y) + |t - mu| exp(-ln b),
//   d nll / d mu = -sign(t - mu) exp(-ln b),   d nll / d ln b = 1 - |t - mu| exp(-ln b),
//   xhat = 2 clamp((sigmoid(mu) - eps) / (1 - 2 eps), 0, 1) - 1 = clamp(2.5 sigmoid(mu) - 1.25, -1, 1).
// An item is V consecutive channels of one pixel (V = 4: 16-byte loads and stores).  One wave of CTAs strides over the
// items; each thread carries its (pixel, group) pair forward by the stride instead of dividing a 64-bit index.
constexpr int LL_THREADS = 256;

__device__ __forceinline__ void ll_one(float mu, float lb, const float* x, float* dmu, float* dlb, float& xh,
                                       float c, float& nll, float& se) {
  xh = fminf(fmaxf(fmaf(2.5f, 1.f / (1.f + expf(-mu)), -1.25f), -1.f), 1.f);
  if (x) {
    const float y = fminf(fmaxf(fmaf(0.4f, *x, 0.5f), 0.1f), 0.9f);
    const float ly = logf(y), l1y = logf(1.f - y);
    const float d = (ly - l1y) - mu;
    const float ib = expf(-lb);
    const float a = fabsf(d) * ib;
    nll += 0.69314718055994531f + lb + (ly + l1y) + a;
    const float e = xh - *x;
    se = fmaf(e, e, se);
    *dmu = d > 0.f ? -c * ib : (d < 0.f ? c * ib : (d == 0.f ? 0.f : d));   // sign(NaN) stays NaN
    *dlb = c * (1.f - a);
  }
}

template <int V>
__global__ void __launch_bounds__(LL_THREADS)
logit_laplace_kernel(const float* __restrict__ stats, const float* __restrict__ target, float* __restrict__ dstats,
                     float* __restrict__ recon, float* __restrict__ partials, long long n_pix, int Cp, float scale) {
  using VT = typename std::conditional<V == 4, float4, float>::type;
  __shared__ float red[2][LL_THREADS / 32];
  const int G = Cp / V;                                     // items per pixel
  const long long start = (long long)blockIdx.x * LL_THREADS + threadIdx.x;
  const long long stride = (long long)gridDim.x * LL_THREADS;
  const long long sp = stride / G;
  const int sg = (int)(stride % G);
  long long p = start / G;
  int g = (int)(start % G);
  float nll = 0.f, se = 0.f;
  for (; p < n_pix;) {
    const long long s0 = p * 2 * Cp + (long long)g * V;     // mu of this item; ln b is Cp further
    const long long i0 = p * Cp + (long long)g * V;
    const VT mu = *reinterpret_cast<const VT*>(stats + s0);
    const VT lb = *reinterpret_cast<const VT*>(stats + s0 + Cp);
    VT xh, dm, dl;
    if (target) {
      const VT x = *reinterpret_cast<const VT*>(target + i0);
      const float* xs = reinterpret_cast<const float*>(&x);
      const float* ms = reinterpret_cast<const float*>(&mu);
      const float* ls = reinterpret_cast<const float*>(&lb);
      float* hs = reinterpret_cast<float*>(&xh);
      float* dms = reinterpret_cast<float*>(&dm);
      float* dls = reinterpret_cast<float*>(&dl);
#pragma unroll
      for (int v = 0; v < V; ++v) ll_one(ms[v], ls[v], xs + v, dms + v, dls + v, hs[v], scale, nll, se);
      *reinterpret_cast<VT*>(dstats + s0) = dm;
      *reinterpret_cast<VT*>(dstats + s0 + Cp) = dl;
    } else {
      const float* ms = reinterpret_cast<const float*>(&mu);
      float* hs = reinterpret_cast<float*>(&xh);
#pragma unroll
      for (int v = 0; v < V; ++v) ll_one(ms[v], 0.f, nullptr, nullptr, nullptr, hs[v], 0.f, nll, se);
    }
    *reinterpret_cast<VT*>(recon + i0) = xh;
    p += sp;
    g += sg;
    if (g >= G) { g -= G; ++p; }
  }
  if (!target) return;
  nll = warp_sum(nll);
  se = warp_sum(se);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { red[0][warp] = nll; red[1][warp] = se; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int w = 0; w < LL_THREADS / 32; ++w) { a += red[0][w]; b += red[1][w]; }
    partials[blockIdx.x] = a * scale;               // per-CTA partials, summed in CTA order by the launcher
    partials[gridDim.x + blockIdx.x] = b * scale;
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
  gumbel_softmax_bwd_kernel<false><<<(rows + 3) / 4, 128, 0, stream>>>(y_soft, dy, dlogits, rows, K, 1.f / tau,
                                                                       nullptr, nullptr, nullptr, 0.f);
  return check_launch("gumbel_softmax_bwd_kernel");
}

extern "C" int db200_gumbel_softmax_bwd_kl(db200_stream_t stream_, const float* y_soft, const float* dy,
                                           const float* logits, const float* lse, const float* ent, float* dlogits,
                                           int rows, int K, float tau, float c) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(y_soft && dy && logits && lse && ent && dlogits && rows > 0 && K > 0 && tau > 0.f && isfinite(c),
                DB200_E_INVALID, "gumbel_softmax_bwd_kl: bad arguments");
  gumbel_softmax_bwd_kernel<true><<<(rows + 3) / 4, 128, 0, stream>>>(y_soft, dy, dlogits, rows, K, 1.f / tau, logits,
                                                                      lse, ent, c);
  return check_launch("gumbel_softmax_bwd_kernel<KL>");
}

// One wave: as many CTAs as fit on the device at once (the shared histogram bounds it), each striding over the rows;
// a second, part-empty wave would leave most SMs idle while it runs.
static int kl_stats_blocks(int rows, int K) {
  int per_sm = 1;   // the four instantiations use the same resources but for the shared histogram
  if (K <= KL_SMEM_HIST_MAX_K)
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, vae_kl_stats_kernel<true, true>, KL_WARPS * 32,
                                                  (size_t)K * sizeof(int));
  else
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, vae_kl_stats_kernel<false, true>, KL_WARPS * 32, 0);
  const long long need = ((long long)rows + KL_WARPS - 1) / KL_WARPS;
  const long long cap = (long long)sm_count() * (per_sm > 0 ? per_sm : 1);
  return (int)(need < cap ? need : cap);
}

extern "C" int64_t db200_vae_kl_stats_workspace_bytes(int rows, int K) {
  return rows > 0 && K > 0 ? (int64_t)kl_stats_blocks(rows, K) * (int64_t)sizeof(float) : 0;
}

extern "C" int db200_vae_kl_stats(db200_stream_t stream_, const float* logits, float* lse, float* ent, int32_t* hist,
                                  float* kl_accum, int rows, int K, float scale, void* workspace,
                                  int64_t workspace_bytes) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(logits && lse && ent && hist && kl_accum && rows > 0 && K > 0 && isfinite(scale), DB200_E_INVALID,
                "vae_kl_stats: bad arguments");
  DB200_REQUIRE(workspace_ok(workspace, workspace_bytes, db200_vae_kl_stats_workspace_bytes(rows, K)),
                DB200_E_INVALID, "vae_kl_stats: needs an aligned workspace of db200_vae_kl_stats_workspace_bytes() bytes");
  const int blocks = kl_stats_blocks(rows, K);
  float* ws = static_cast<float*>(workspace);
  const bool vec4 = K % 4 == 0 && aligned16(logits);
  const size_t smem = K <= KL_SMEM_HIST_MAX_K ? (size_t)K * sizeof(int) : 0;
  auto kernel = K <= KL_SMEM_HIST_MAX_K ? (vec4 ? vae_kl_stats_kernel<true, true> : vae_kl_stats_kernel<true, false>)
                                        : (vec4 ? vae_kl_stats_kernel<false, true> : vae_kl_stats_kernel<false, false>);
  kernel<<<blocks, KL_WARPS * 32, smem, stream>>>(logits, lse, ent, hist, ws, rows, K, (float)K, scale);
  const int rc = check_launch("vae_kl_stats_kernel");
  if (rc != DB200_OK) return rc;
  return reduce_rows_add(stream, ws, blocks, 1, kl_accum);
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

// One wave: as many CTAs as fit on the device at once, each striding over the items, but no more than the items need.
static int logit_laplace_blocks(long long n_pix, int Cp) {
  int per_sm = 1;   // both instantiations: 256 threads, the same small static shared memory
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, logit_laplace_kernel<1>, LL_THREADS, 0);
  const long long items = n_pix * (Cp % 4 == 0 ? Cp / 4 : Cp);
  const long long need = (items + LL_THREADS - 1) / LL_THREADS;
  const long long cap = (long long)sm_count() * (per_sm > 0 ? per_sm : 1);
  return (int)(need < cap ? need : cap);
}

extern "C" int64_t db200_logit_laplace_workspace_bytes(int64_t n_pix, int Cp) {
  return n_pix > 0 && Cp > 0 ? 2 * (int64_t)logit_laplace_blocks(n_pix, Cp) * (int64_t)sizeof(float) : 0;
}

extern "C" int db200_logit_laplace_fwd_bwd(db200_stream_t stream_, const float* stats, const float* target,
                                           float* dstats, float* recon_out, float* nll_accum, float* mse_accum,
                                           int64_t n_pix, int Cp, float scale, void* workspace,
                                           int64_t workspace_bytes) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(stats && recon_out && n_pix > 0 && Cp > 0 && n_pix <= INT64_MAX / (2 * (int64_t)Cp) &&
                isfinite(scale), DB200_E_INVALID, "logit_laplace: bad arguments");
  DB200_REQUIRE(!target || (dstats && nll_accum && mse_accum), DB200_E_INVALID,
                "logit_laplace: a target needs dstats, nll_accum and mse_accum");
  const int blocks = logit_laplace_blocks(n_pix, Cp);
  DB200_REQUIRE(!target || workspace_ok(workspace, workspace_bytes, 2 * (int64_t)blocks * (int64_t)sizeof(float)),
                DB200_E_INVALID,
                "logit_laplace: needs an aligned workspace of db200_logit_laplace_workspace_bytes() bytes");
  float* ws = static_cast<float*>(workspace);
  const bool vec4 = Cp % 4 == 0 && aligned16(stats) && aligned16(recon_out) &&
                    (!target || (aligned16(target) && aligned16(dstats)));
  if (vec4)
    logit_laplace_kernel<4><<<blocks, LL_THREADS, 0, stream>>>(stats, target, dstats, recon_out, ws, n_pix, Cp,
                                                              scale);
  else
    logit_laplace_kernel<1><<<blocks, LL_THREADS, 0, stream>>>(stats, target, dstats, recon_out, ws, n_pix, Cp,
                                                              scale);
  const int rc = check_launch("logit_laplace_kernel");
  if (rc != DB200_OK || !target) return rc;
  const int rc2 = reduce_rows_add(stream, ws, blocks, 1, nll_accum);
  if (rc2 != DB200_OK) return rc2;
  return reduce_rows_add(stream, ws + blocks, blocks, 1, mse_accum);
}
