// K9 / K10 — global gradient norm and fused multi-tensor Adam over FLAT parameter / state / gradient buffers.
// Pure HBM-bound streaming kernels: 4 B/param read for the norm; 16 B read + 12 B (+2 B bf16 shadow) written per
// parameter for Adam.  No host synchronisation: the clip factor is computed on the device from the norm scalar.
//
// Reference: clip_by_global_norm src/optimizers.py:11-16; mtf AdamWeightDecayOptimizer restated in-tree at
// src/optimizers.py:128-172 (no bias correction, eps 1e-6); tf.train.AdamOptimizer (bias-corrected, eps 1e-8) as
// used for the VAE at src/model_fns_tf.py:58-66.
#include "common.cuh"
#include "ptx.cuh"

namespace db200 {

__global__ void __launch_bounds__(256) sqnorm_kernel(const float* __restrict__ g, size_t n, float* __restrict__ out) {
  __shared__ float red[8];
  const size_t nv = n >> 2;
  float acc = 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const float t = g[(nv << 2) + threadIdx.x];
    acc += t * t;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w];
    out[blockIdx.x] = s;  // one partial per block, summed in block order by reduce_rows_add
  }
}

struct AdamArgs {
  float lr, beta1, beta2, eps, wd, clip, grad_scale;
  int bias_correction;
  float lr_t;  // lr * sqrt(1-b2^t) / (1-b1^t) when bias_correction
  int zero_grad;  // write 0 back over the gradient once it has been consumed (saves next step's 4 B/param memset pass)
};

__device__ __forceinline__ float adam_one(float& p, float& m, float& v, float g, const AdamArgs& a, float gmul) {
  const float gs = g * gmul;
  m = a.beta1 * m + (1.f - a.beta1) * gs;
  v = a.beta2 * v + (1.f - a.beta2) * gs * gs;
  if (a.bias_correction) {
    p -= a.lr_t * m / (sqrtf(v) + a.eps);
  } else {
    float upd = m / (sqrtf(v) + a.eps);
    if (a.wd != 0.f) upd += a.wd * p;
    p -= a.lr * upd;
  }
  return p;
}

__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v, float* __restrict__ g,
            bf16* __restrict__ p16, size_t n, AdamArgs a, const float* __restrict__ gnorm_sq) {
  float gmul = a.grad_scale;
  if (gnorm_sq != nullptr && a.clip > 0.f) {
    const float gn = sqrtf(*gnorm_sq) * a.grad_scale;  // norm of the scaled gradient
    gmul *= a.clip / fmaxf(gn, a.clip);
  }
  const size_t nv = n >> 2;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
    float4 pp = reinterpret_cast<float4*>(p)[i];
    float4 mm = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
    adam_one(pp.x, mm.x, vv.x, gg.x, a, gmul);
    adam_one(pp.y, mm.y, vv.y, gg.y, a, gmul);
    adam_one(pp.z, mm.z, vv.z, gg.z, a, gmul);
    adam_one(pp.w, mm.w, vv.w, gg.w, a, gmul);
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(m)[i] = mm;
    reinterpret_cast<float4*>(v)[i] = vv;
    if (a.zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p16) {
      uint2 o;
      o.x = pack_bf16x2(pp.x, pp.y);
      o.y = pack_bf16x2(pp.z, pp.w);
      reinterpret_cast<uint2*>(p16)[i] = o;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const size_t i = (nv << 2) + threadIdx.x;
    float pp = p[i], mm = m[i], vv = v[i];
    adam_one(pp, mm, vv, g[i], a, gmul);
    p[i] = pp; m[i] = mm; v[i] = vv;
    if (a.zero_grad) g[i] = 0.f;
    if (p16) p16[i] = __float2bfloat16(pp);
  }
}

}  // namespace db200

using namespace db200;

static size_t sqnorm_blocks(size_t n) {
  size_t blocks = (n / 4 + 255) / 256;
  const size_t cap = (size_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  return blocks < 1 ? 1 : blocks;
}

extern "C" int64_t db200_sqnorm_workspace_bytes(size_t n) { return (int64_t)(sqnorm_blocks(n) * sizeof(float)); }

extern "C" int db200_sqnorm_f32(db200_stream_t stream_, const float* g, size_t n, float* out_accum, void* workspace,
                                int64_t workspace_bytes) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (n == 0) return DB200_OK;
  DB200_REQUIRE(g && out_accum && aligned16(g), DB200_E_ALIGN, "sqnorm: NULL or unaligned pointer");
  const size_t blocks = sqnorm_blocks(n);
  DB200_REQUIRE(workspace_ok(workspace, workspace_bytes, (int64_t)(blocks * sizeof(float))), DB200_E_INVALID,
                "sqnorm: needs an aligned workspace of db200_sqnorm_workspace_bytes() bytes");
  float* ws = static_cast<float*>(workspace);
  sqnorm_kernel<<<(int)blocks, 256, 0, stream>>>(g, n, ws);
  const int rc = check_launch("sqnorm_kernel");
  if (rc != DB200_OK) return rc;
  return reduce_rows_add(stream, ws, (int)blocks, 1, out_accum);
}

extern "C" int db200_adam_step(db200_stream_t stream_, float* p, float* m, float* v, float* g, void* p_bf16,
                               size_t n, float lr, float beta1, float beta2, float eps, float weight_decay,
                               const float* gnorm_sq, float clip, float grad_scale, int bias_correction, int step,
                               int zero_grad) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (n == 0) return DB200_OK;
  DB200_REQUIRE(p && m && v && g, DB200_E_INVALID, "adam: NULL pointer");
  DB200_REQUIRE(aligned16(p) && aligned16(m) && aligned16(v) && aligned16(g) &&
                    (reinterpret_cast<uintptr_t>(p_bf16) & 7u) == 0,
                DB200_E_ALIGN, "adam: buffers must be 16-byte aligned (bf16 shadow 8-byte)");
  DB200_REQUIRE(!bias_correction || step >= 1, DB200_E_INVALID, "adam: bias_correction needs step >= 1 (got %d)",
                step);
  AdamArgs a;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.wd = weight_decay; a.clip = clip;
  a.grad_scale = grad_scale;
  a.bias_correction = bias_correction;
  a.zero_grad = zero_grad;
  a.lr_t = lr;
  if (bias_correction) {
    const double b1t = 1.0 - pow((double)beta1, (double)step), b2t = 1.0 - pow((double)beta2, (double)step);
    a.lr_t = (float)((double)lr * sqrt(b2t) / b1t);
  }
  size_t blocks = (n / 4 + 255) / 256;
  const size_t cap = (size_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  adam_kernel<<<(int)blocks, 256, 0, stream>>>(p, m, v, g, (bf16*)p_bf16, n, a, gnorm_sq);
  return check_launch("adam_kernel");
}
