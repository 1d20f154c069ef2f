// K1 / K2 and the small HBM-bound helpers: embedding gather/scatter, LayerNorm fwd/bwd, column sums, casts,
// cross-entropy finish.  All are coalesced 16-byte-vectorised kernels with warp-shuffle row reductions; none has
// data reuse worth staging in shared memory.  Roofline: HBM.
//
// Reference: src/dalle_mtf/models.py:186-219 (embedding), :373-389 + src/dalle_mtf/layers.py:30-33 (LayerNorm),
//            :348-359 (loss reduction).
#include "common.cuh"
#include "philox.cuh"
#include "ptx.cuh"

namespace db200 {

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  return u;
}

// ------------------------------------------------------------------------------------------------ embedding
__global__ void embed_fwd_kernel(const int* __restrict__ ids, const bf16* __restrict__ wte,
                                 const bf16* __restrict__ wpe, bf16* __restrict__ out, int T, int S, int d, int V) {
  const int vec_per_row = d >> 3;
  const long long total = (long long)T * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / vec_per_row);
    const int c = (int)(i - (long long)t * vec_per_row) << 3;
    int id = ids[t];
    id = id < 0 ? 0 : (id >= V ? V - 1 : id);  // ids are validated on the host; clamp instead of faulting
    const int s = t % S;
    float a[8], b[8];
    unpack8(*reinterpret_cast<const uint4*>(wte + (long long)id * d + c), a);
    unpack8(*reinterpret_cast<const uint4*>(wpe + (long long)s * d + c), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    *reinterpret_cast<uint4*>(out + (long long)t * d + c) = pack8(a);
  }
}

// 8 keep multipliers (keep ? scale : 0) of columns c .. c + 7 of row r of an elementwise mask over [rows][cols]
__device__ __forceinline__ void dropout_mul8(const db200_dropout& dr, long long r, int cols, int c, float* m) {
  const uint64_t n0 = dropout_elem_block(dr, r, cols, c);
  const uint4 a = dropout_block(dr, n0), b = dropout_block(dr, n0 + 1);
  m[0] = dropout_mul(dr, a.x); m[1] = dropout_mul(dr, a.y); m[2] = dropout_mul(dr, a.z); m[3] = dropout_mul(dr, a.w);
  m[4] = dropout_mul(dr, b.x); m[5] = dropout_mul(dr, b.y); m[6] = dropout_mul(dr, b.z); m[7] = dropout_mul(dr, b.w);
}

// embedding dropout (src/dalle_mtf/models.py:198-200, 215-217): out = wte[id] * keep_wte * scale + wpe[s] * keep_wpe *
// scale; the wte mask is over the [T][d] gathered rows, the wpe mask over [S][d] (shared by the batch)
__global__ void embed_fwd_drop_kernel(const int* __restrict__ ids, const bf16* __restrict__ wte,
                                      const bf16* __restrict__ wpe, bf16* __restrict__ out, int T, int S, int d, int V,
                                      const db200_dropout dw, const db200_dropout dp) {
  const int vec_per_row = d >> 3;
  const long long total = (long long)T * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / vec_per_row);
    const int c = (int)(i - (long long)t * vec_per_row) << 3;
    int id = ids[t];
    id = id < 0 ? 0 : (id >= V ? V - 1 : id);
    const int s = t % S;
    float a[8], b[8], ma[8], mb[8];
    unpack8(*reinterpret_cast<const uint4*>(wte + (long long)id * d + c), a);
    unpack8(*reinterpret_cast<const uint4*>(wpe + (long long)s * d + c), b);
    dropout_mul8(dw, t, d, c, ma);
    dropout_mul8(dp, s, d, c, mb);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = a[j] * ma[j] + b[j] * mb[j];
    *reinterpret_cast<uint4*>(out + (long long)t * d + c) = pack8(a);
  }
}

// dwte[ids[t]] += dx[t].  A thread owns 8 columns of a strip of EMB_STRIP consecutive tokens and merges RUNS of equal
// ids in registers before touching memory: captions are right-padded with one id (src/input_fns.py:32-38), so the
// ~220 consecutive padding positions of every sequence collapse into one reduction per strip instead of 220 serialised
// reductions on the same row (same-address reductions serialise in L2).  Strips of different tokens meet on the same
// row in no fixed order, so the run sums go into a 64-bit fixed-point accumulator in the caller's workspace (cleared
// on the stream first; integer addition is associative: the result does not depend on that order) that
// embed_fixed_flush_kernel then adds to dwte.
constexpr double EMB_FIX_SCALE = 1099511627776.0;  // 2^40: resolution 9.1e-13, magnitude up to 8.4e6
__device__ __forceinline__ void fixed_add(unsigned long long* dst, float v) {
  atomicAdd(dst, static_cast<unsigned long long>(__double2ll_rn(static_cast<double>(v) * EMB_FIX_SCALE)));
}
// DROP: dx[t] is multiplied by the wte keep mask first.  SCALE (the stable embedding's gradient shrink): then by
// alpha, rounded on its own in fp32 before it is summed.
constexpr int EMB_STRIP = 32;
template <bool DROP, bool SCALE = false>
__global__ void __launch_bounds__(256)
embed_bwd_wte_kernel(const int* __restrict__ ids, const bf16* __restrict__ dx, unsigned long long* __restrict__ acc64,
                     int T, int d, int V, const db200_dropout dw, float alpha = 1.f) {
  const int vec_per_row = d >> 3;
  const long long total = (long long)((T + EMB_STRIP - 1) / EMB_STRIP) * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int strip = (int)(i / vec_per_row);
    const int c = (int)(i - (long long)strip * vec_per_row) << 3;
    const int t0 = strip * EMB_STRIP, t1 = min(T, t0 + EMB_STRIP);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int cur = -1;
    auto flush = [&]() {
      if (cur >= 0 && cur < V) {
        unsigned long long* dst = acc64 + (long long)cur * d + c;
#pragma unroll
        for (int j = 0; j < 8; ++j) fixed_add(dst + j, acc[j]);
      }
    };
    for (int t = t0; t < t1; ++t) {
      const int id = ids[t];
      if (id != cur) {
        flush();
        cur = id;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
      }
      float g[8];
      unpack8(*reinterpret_cast<const uint4*>(dx + (long long)t * d + c), g);
      if constexpr (DROP) {
        float m[8];
        dropout_mul8(dw, t, d, c, m);
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] *= m[j];
      }
      if constexpr (SCALE) {
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] = __fmul_rn(g[j], alpha);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += g[j];
    }
    flush();
  }
}

// dwte += acc64 / 2^40 where acc64 is non-zero
__global__ void __launch_bounds__(256)
embed_fixed_flush_kernel(const unsigned long long* __restrict__ acc64, float* __restrict__ dwte, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long v = static_cast<long long>(acc64[i]);
    if (v != 0) {
      dwte[i] += static_cast<float>(static_cast<double>(v) * (1.0 / EMB_FIX_SCALE));
    }
  }
}

// one thread owns (s, 8 columns): dwpe[s][c..c+8) += sum_b dx[b][s][c..c+8)   (DROP: times the wpe keep mask of s,
// which every sequence shares; SCALE: each dx element times alpha, rounded on its own, before it is summed)
template <bool DROP, bool SCALE = false>
__global__ void embed_bwd_wpe_kernel(const bf16* __restrict__ dx, float* __restrict__ dwpe, int B, int S, int d,
                                     const db200_dropout dp, float alpha = 1.f) {
  const int vec_per_row = d >> 3;
  const int total = S * vec_per_row;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int s = i / vec_per_row;
  const int c = (i - s * vec_per_row) << 3;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int b = 0; b < B; ++b) {
    float g[8];
    unpack8(*reinterpret_cast<const uint4*>(dx + ((long long)b * S + s) * d + c), g);
    if constexpr (SCALE) {
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = __fmul_rn(g[j], alpha);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += g[j];
  }
  if constexpr (DROP) {
    float m[8];
    dropout_mul8(dp, s, d, c, m);
    // rounded on its own (__fmul_rn is never contracted with the add below into an fma): the call adds one fully
    // formed contribution, so W ranks summed in rank order equal one rank running the same rows as W micro-batches
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = __fmul_rn(acc[j], m[j]);
  }
  float* dst = dwpe + (long long)s * d + c;
#pragma unroll
  for (int j = 0; j < 8; ++j) dst[j] += acc[j];
}

// labels[b][t] = ids[b][t+1] for t < S-1, labels[b][S-1] = eos      (src/dalle_mtf/models.py:407-410)
__global__ void shift_labels_kernel(const int* __restrict__ ids, int* __restrict__ labels, int B, int S, int eos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * S) return;
  const int t = i % S;
  labels[i] = (t == S - 1) ? eos : ids[i + 1];
}

// tokens[b][:] = concat(text[b][:Tt], image_idx[b][:Ti] + offset)       (src/model_fns.py:117-122)
__global__ void assemble_tokens_kernel(const int* __restrict__ text, const int* __restrict__ img, int* __restrict__ out,
                                       int B, int Tt, int Ti, int offset) {
  const int S = Tt + Ti;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * S) return;
  const int b = i / S, t = i - b * S;
  out[i] = t < Tt ? text[b * Tt + t] : img[b * Ti + (t - Tt)] + offset;
}

// One token of the assembly with caption dropout or per-position pads.  DROP: caption dropout, row b's text positions
// all become a pad when the Philox word of global sequence index e = dr.row0 + b (elementwise layout with cols = 1:
// block e >> 2, word e & 3) is below dr.threshold.  PER_POS: the pad of text position t is pad_base + t, and a caption
// id equal to `pad` becomes that per-position pad too (DALL-E's separate padding token for each text position); without
// it a dropped caption is `pad` everywhere and caption ids pass through unchanged.
template <bool DROP, bool PER_POS>
__device__ __forceinline__ void assemble_one(const int* __restrict__ text, const int* __restrict__ img,
                                             int* __restrict__ out, int B, int Tt, int Ti, int offset, int pad,
                                             int pad_base, const db200_dropout& dr) {
  const int S = Tt + Ti;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * S) return;
  const int b = i / S, t = i - b * S;
  if (t < Tt) {
    bool dropped = false;
    if constexpr (DROP) {
      const uint4 words = dropout_block(dr, dropout_elem_block(dr, b, 1, 0));
      dropped = uint4_word(words, (int)((dr.row0 + b) & 3)) < dr.threshold;
    }
    if constexpr (PER_POS) {
      const int id = text[b * Tt + t];
      out[i] = (dropped || id == pad) ? pad_base + t : id;
    } else {
      out[i] = dropped ? pad : text[b * Tt + t];
    }
  } else {
    out[i] = img[b * Ti + (t - Tt)] + offset;
  }
}

// assemble_tokens_kernel with caption dropout
__global__ void assemble_tokens_drop_kernel(const int* __restrict__ text, const int* __restrict__ img,
                                            int* __restrict__ out, int B, int Tt, int Ti, int offset, int pad,
                                            const db200_dropout dr) {
  assemble_one<true, false>(text, img, out, B, Tt, Ti, offset, pad, 0, dr);
}

// the same with per-position pads (DROP: and caption dropout)
template <bool DROP>
__global__ void assemble_tokens_pp_kernel(const int* __restrict__ text, const int* __restrict__ img,
                                          int* __restrict__ out, int B, int Tt, int Ti, int offset, int pad,
                                          int pad_base, const db200_dropout dr) {
  assemble_one<DROP, true>(text, img, out, B, Tt, Ti, offset, pad, pad_base, dr);
}

// ------------------------------------------------------------------------------------------------ row / column positions
// pos[p] = wpe[p] for p < TL, pos[TL + r W + c] = bf16_rn(float(row[r]) + float(col[c])): the [S][d] bf16 table the
// embedding kernels read in place of an absolute wpe.  One thread per (position, 8 columns), 16-byte loads and stores.
__global__ void __launch_bounds__(256)
pos_compose_kernel(const bf16* __restrict__ wpe, const bf16* __restrict__ row, const bf16* __restrict__ col,
                   bf16* __restrict__ out, int TL, int W, int d) {
  const int vec_per_row = d >> 3;
  const long long total = (long long)(TL + W * W) * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(i / vec_per_row);
    const int c = (int)(i - (long long)p * vec_per_row) << 3;
    uint4 v;
    if (p < TL) {
      v = *reinterpret_cast<const uint4*>(wpe + (long long)p * d + c);
    } else {
      const int r = (p - TL) / W, k = (p - TL) - r * W;
      float a[8], b[8];
      unpack8(*reinterpret_cast<const uint4*>(row + (long long)r * d + c), a);
      unpack8(*reinterpret_cast<const uint4*>(col + (long long)k * d + c), b);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += b[j];
      v = pack8(a);
    }
    *reinterpret_cast<uint4*>(out + (long long)p * d + c) = v;
  }
}

// The transpose of pos_compose on fp32 gradients: dwpe[p] += dpos[p] (p < TL), drow[r] += sum_c dpos[TL + r W + c] with c
// ascending, dcol[c] += sum_r dpos[TL + r W + c] with r ascending.  One thread per (output row, 8 columns): every sum
// runs in registers in that fixed order and is added to the gradient once, so the result is bit-reproducible and a call
// adds one fully formed contribution (W ranks summed in rank order equal one rank running W micro-batches).
__global__ void __launch_bounds__(256)
pos_fold_kernel(const float* __restrict__ dpos, float* __restrict__ dwpe, float* __restrict__ drow,
                float* __restrict__ dcol, int TL, int W, int d) {
  const int vec_per_row = d >> 3;
  const long long total = (long long)(TL + 2 * W) * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)(i / vec_per_row);
    const int c = (int)(i - (long long)o * vec_per_row) << 3;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float* dst;
    long long p0, stride;
    int n;
    if (o < TL) {
      dst = dwpe + (long long)o * d; p0 = o; stride = 0; n = 1;
    } else if (o < TL + W) {
      const int r = o - TL;
      dst = drow + (long long)r * d; p0 = TL + (long long)r * W; stride = 1; n = W;
    } else {
      const int k = o - TL - W;
      dst = dcol + (long long)k * d; p0 = TL + k; stride = W; n = W;
    }
    for (int j = 0; j < n; ++j) {
      const float* src = dpos + (p0 + j * stride) * d + c;
      const float4 u = *reinterpret_cast<const float4*>(src), w = *reinterpret_cast<const float4*>(src + 4);
      acc[0] += u.x; acc[1] += u.y; acc[2] += u.z; acc[3] += u.w;
      acc[4] += w.x; acc[5] += w.y; acc[6] += w.z; acc[7] += w.w;
    }
    float4* q = reinterpret_cast<float4*>(dst + c);
    float4 u = q[0], w = q[1];
    u.x += acc[0]; u.y += acc[1]; u.z += acc[2]; u.w += acc[3];
    w.x += acc[4]; w.y += acc[5]; w.z += acc[6]; w.w += acc[7];
    q[0] = u; q[1] = w;
  }
}

// ------------------------------------------------------------------------------------------------ LayerNorm
// o[j] = r[j] + o[j] for the 8 bf16 residual values at r (the sandwich LayerNorm's residual add, in fp32)
__device__ __forceinline__ void ln_add_res8(const bf16* r, float* o) {
  float rv[8];
  unpack8(*reinterpret_cast<const uint4*>(r), rv);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = rv[j] + o[j];
}
// o[j] = r[j] + s[j] * o[j] (LayerScale on the sandwich LayerNorm's output, in fp32) for the 8 columns at r / s
__device__ __forceinline__ void ln_add_scaled_res8(const bf16* r, const float* s, float* o) {
  float rv[8];
  unpack8(*reinterpret_cast<const uint4*>(r), rv);
  const float4 s0 = *reinterpret_cast<const float4*>(s), s1 = *reinterpret_cast<const float4*>(s + 4);
  const float ss[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = rv[j] + ss[j] * o[j];
}

// One warp per row; the row lives in registers (NCH 16-byte chunks per lane, d = NCH * 256).
// RES (sandwich LayerNorm): y = bf16(res + (x - mean) * rstd * g + b), one rounding; the statistics are the same
// instructions as without it.  `res` is a trailing parameter so that the RES = false kernels keep their code.
// SCALE (with RES, LayerScale): y = bf16(res + scale * ((x - mean) * rstd * g + b)), one rounding.
// DIVMAX (the stable final LayerNorm's DivideMax): the row is first divided by its maximum m (written to m_out), u =
// x / m in fp32 (IEEE division), and the LayerNorm is that of u.
template <int NCH, bool RES = false, bool SCALE = false, bool DIVMAX = false>
__global__ void __launch_bounds__(128)
layernorm_fwd_kernel(const bf16* __restrict__ x, const float* __restrict__ g, const float* __restrict__ b,
                     bf16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows,
                     float eps, const bf16* __restrict__ res = nullptr, const float* __restrict__ scale = nullptr,
                     float* __restrict__ m_out = nullptr) {
  constexpr int d = NCH * 256;
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const bf16* xr = x + (long long)row * d;
  float v[NCH][8];
  float sum = 0.f;
  if constexpr (DIVMAX) {
    float mx = -INFINITY;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      unpack8(*reinterpret_cast<const uint4*>(xr + (c * 32 + lane) * 8), v[c]);
#pragma unroll
      for (int j = 0; j < 8; ++j) mx = fmaxf(mx, v[c][j]);
    }
    mx = warp_max(mx);
    if (lane == 0) m_out[row] = mx;
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[c][j] = __fdiv_rn(v[c][j], mx);
        sum += v[c][j];
      }
  } else {
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      unpack8(*reinterpret_cast<const uint4*>(xr + (c * 32 + lane) * 8), v[c]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[c][j];
    }
  }
  const float mean = warp_sum(sum) * (1.f / d);
  float sq = 0.f;
#pragma unroll
  for (int c = 0; c < NCH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float t = v[c][j] - mean;
      sq += t * t;
    }
  const float rstd = rsqrtf(warp_sum(sq) * (1.f / d) + eps);
  if (lane == 0) {
    mean_out[row] = mean;
    rstd_out[row] = rstd;
  }
  bf16* yr = y + (long long)row * d;
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int col = (c * 32 + lane) * 8;
    const float4 g0 = *reinterpret_cast<const float4*>(g + col), g1 = *reinterpret_cast<const float4*>(g + col + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(b + col), b1 = *reinterpret_cast<const float4*>(b + col + 4);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = (v[c][j] - mean) * rstd * gg[j] + bb[j];
    if constexpr (SCALE) ln_add_scaled_res8(res + (long long)row * d + col, scale + col, o);
    else if constexpr (RES) ln_add_res8(res + (long long)row * d + col, o);
    *reinterpret_cast<uint4*>(yr + col) = pack8(o);
  }
}

// store 8 columns of dx; DROP: also dxm = dx * keep * scale (mask of row `row` over [rows][d]).  The column sum adx
// takes the values exactly as stored (bf16-rounded), of dxm when DROP and of dx otherwise, like a separate column-sum
// pass would.
template <bool DROP>
__device__ __forceinline__ void ln_bwd_store8(const float* o, bf16* dx, bf16* dxm, long long row, int d, int col,
                                              bool dxsum, const db200_dropout& dr, float* adx) {
  const uint4 packed = pack8(o);
  *reinterpret_cast<uint4*>(dx + row * d + col) = packed;
  float ro[8];
  unpack8(packed, ro);
  if constexpr (DROP) {
    float m[8];
    dropout_mul8(dr, row, d, col, m);
#pragma unroll
    for (int j = 0; j < 8; ++j) ro[j] *= m[j];
    const uint4 pm = pack8(ro);
    *reinterpret_cast<uint4*>(dxm + row * d + col) = pm;
    unpack8(pm, ro);
  }
  if (dxsum) {
#pragma unroll
    for (int j = 0; j < 8; ++j) adx[j] += ro[j];
  }
}

// Each warp walks rows with a grid stride, keeps per-lane partial dg/db in registers, then one block-level
// reduction through shared memory and one partial row of dg / db (/ dxsum) per block, summed in block order afterwards.
// DIVMAX (the DivideMax LayerNorm): the normalised row is u = x / m with the row's m_in (the same IEEE division as
// the forward) and the gradient is divided by m, dx = LN'(u)^T dy / m, before the residual term and the store.
template <int NCH, bool DROP, bool DIVMAX = false>
__global__ void __launch_bounds__(128)
layernorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, const float* __restrict__ g,
                     const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                     const bf16* __restrict__ dres, bf16* __restrict__ dx, float* __restrict__ dg,
                     float* __restrict__ db, float* __restrict__ dxsum, int rows, bf16* __restrict__ dxm,
                     const db200_dropout dr, const float* __restrict__ m_in = nullptr) {
  constexpr int d = NCH * 256;
  __shared__ float red[4][d];  // NCH <= 8 -> <= 32 KiB
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  float gg[NCH][8];
  float adg[NCH][8], adb[NCH][8], adx[NCH][8];
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int col = (c * 32 + lane) * 8;
    const float4 g0 = *reinterpret_cast<const float4*>(g + col), g1 = *reinterpret_cast<const float4*>(g + col + 4);
    gg[c][0] = g0.x; gg[c][1] = g0.y; gg[c][2] = g0.z; gg[c][3] = g0.w;
    gg[c][4] = g1.x; gg[c][5] = g1.y; gg[c][6] = g1.z; gg[c][7] = g1.w;
#pragma unroll
    for (int j = 0; j < 8; ++j) adg[c][j] = adb[c][j] = adx[c][j] = 0.f;
  }
  for (int row = blockIdx.x * 4 + warp; row < rows; row += gridDim.x * 4) {
    const float mean = mean_in[row], rstd = rstd_in[row];
    const bf16* xr = x + (long long)row * d;
    const bf16* dyr = dy + (long long)row * d;
    float xh[NCH][8], dg_[NCH][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col = (c * 32 + lane) * 8;
      float xv[8], dv[8];
      unpack8(*reinterpret_cast<const uint4*>(xr + col), xv);
      unpack8(*reinterpret_cast<const uint4*>(dyr + col), dv);
      if constexpr (DIVMAX) {
#pragma unroll
        for (int j = 0; j < 8; ++j) xv[j] = __fdiv_rn(xv[j], m_in[row]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float h = (xv[j] - mean) * rstd;
        const float t = dv[j] * gg[c][j];
        xh[c][j] = h;
        dg_[c][j] = t;
        s1 += t;
        s2 += t * h;
        adg[c][j] += dv[j] * h;
        adb[c][j] += dv[j];
      }
    }
    const float c1 = warp_sum(s1) * (1.f / d), c2 = warp_sum(s2) * (1.f / d);
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col = (c * 32 + lane) * 8;
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (dg_[c][j] - c1 - xh[c][j] * c2) * rstd;
      if constexpr (DIVMAX) {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = __fdiv_rn(o[j], m_in[row]);
      }
      if (dres) {
        float r[8];
        unpack8(*reinterpret_cast<const uint4*>(dres + (long long)row * d + col), r);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += r[j];
      }
      ln_bwd_store8<DROP>(o, dx, dxm, row, d, col, dxsum != nullptr, dr, adx[c]);
    }
  }
  // block reduction of dg, then db (then dxsum)
  const int npass = dxsum ? 3 : 2;
#pragma unroll 1
  for (int pass = 0; pass < npass; ++pass) {
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j)
        red[warp][(c * 32 + lane) * 8 + j] = pass == 0 ? adg[c][j] : (pass == 1 ? adb[c][j] : adx[c][j]);
    __syncthreads();
    float* dst = (pass == 0 ? dg : (pass == 1 ? db : dxsum)) + (long long)blockIdx.x * d;  // this block's partial row
    for (int col = threadIdx.x; col < d; col += 128)
      dst[col] = red[0][col] + red[1][col] + red[2][col] + red[3][col];
    __syncthreads();
  }
}

// Wide rows (d = 4096, the 12 B configuration): ONE CTA of 128 threads per row, thread t owns columns
// {(c*128 + t)*8 .. +7 : c < NCW} (16-byte accesses, 2 KiB contiguous per c across the CTA).  Row statistics go through
// a two-level (warp shuffle + 4-float shared) reduction; in backward every thread owns its columns for the whole row
// walk, so dgamma / dbeta / dxsum need no cross-thread reduction at all: one partial row per CTA at the end.
__device__ __forceinline__ float2 block128_sum2(float a, float b, float* red /*[8]*/) {
  a = warp_sum(a);
  b = warp_sum(b);
  const int warp = threadIdx.x >> 5;
  __syncthreads();  // previous use of `red` is over
  if ((threadIdx.x & 31) == 0) { red[warp] = a; red[4 + warp] = b; }
  __syncthreads();
  return make_float2(red[0] + red[1] + red[2] + red[3], red[4] + red[5] + red[6] + red[7]);
}
__device__ __forceinline__ float block128_max(float a, float* red /*[8]*/) {
  a = warp_max(a);
  __syncthreads();  // previous use of `red` is over
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  return fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
}

template <int NCW, bool RES = false, bool SCALE = false, bool DIVMAX = false>
__global__ void __launch_bounds__(128)
layernorm_fwd_wide_kernel(const bf16* __restrict__ x, const float* __restrict__ g, const float* __restrict__ b,
                          bf16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows,
                          float eps, const bf16* __restrict__ res = nullptr,
                          const float* __restrict__ scale = nullptr, float* __restrict__ m_out = nullptr) {
  constexpr int d = NCW * 1024;
  __shared__ float red[8];
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const bf16* xr = x + (long long)row * d;
    float v[NCW][8];
    float sum = 0.f;
    if constexpr (DIVMAX) {
      float mx = -INFINITY;
#pragma unroll
      for (int c = 0; c < NCW; ++c) {
        unpack8(*reinterpret_cast<const uint4*>(xr + (c * 128 + threadIdx.x) * 8), v[c]);
#pragma unroll
        for (int j = 0; j < 8; ++j) mx = fmaxf(mx, v[c][j]);
      }
      mx = block128_max(mx, red);
      if (threadIdx.x == 0) m_out[row] = mx;
#pragma unroll
      for (int c = 0; c < NCW; ++c)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          v[c][j] = __fdiv_rn(v[c][j], mx);
          sum += v[c][j];
        }
    } else {
#pragma unroll
      for (int c = 0; c < NCW; ++c) {
        unpack8(*reinterpret_cast<const uint4*>(xr + (c * 128 + threadIdx.x) * 8), v[c]);
#pragma unroll
        for (int j = 0; j < 8; ++j) sum += v[c][j];
      }
    }
    const float mean = block128_sum2(sum, 0.f, red).x * (1.f / d);
    float sq = 0.f;
#pragma unroll
    for (int c = 0; c < NCW; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float t = v[c][j] - mean;
        sq += t * t;
      }
    const float rstd = rsqrtf(block128_sum2(sq, 0.f, red).x * (1.f / d) + eps);
    if (threadIdx.x == 0) {
      mean_out[row] = mean;
      rstd_out[row] = rstd;
    }
    bf16* yr = y + (long long)row * d;
#pragma unroll
    for (int c = 0; c < NCW; ++c) {
      const int col = (c * 128 + threadIdx.x) * 8;
      const float4 g0 = *reinterpret_cast<const float4*>(g + col), g1 = *reinterpret_cast<const float4*>(g + col + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(b + col), b1 = *reinterpret_cast<const float4*>(b + col + 4);
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[c][j] - mean) * rstd * gg[j] + bb[j];
      if constexpr (SCALE) ln_add_scaled_res8(res + (long long)row * d + col, scale + col, o);
      else if constexpr (RES) ln_add_res8(res + (long long)row * d + col, o);
      *reinterpret_cast<uint4*>(yr + col) = pack8(o);
    }
  }
}

template <int NCW, bool DROP, bool DIVMAX = false>
__global__ void __launch_bounds__(128)
layernorm_bwd_wide_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, const float* __restrict__ g,
                          const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                          const bf16* __restrict__ dres, bf16* __restrict__ dx, float* __restrict__ dg,
                          float* __restrict__ db, float* __restrict__ dxsum, int rows, bf16* __restrict__ dxm,
                          const db200_dropout dr, const float* __restrict__ m_in = nullptr) {
  constexpr int d = NCW * 1024;
  __shared__ float red[8];
  float gg[NCW][8], adg[NCW][8], adb[NCW][8], adx[NCW][8];
#pragma unroll
  for (int c = 0; c < NCW; ++c) {
    const int col = (c * 128 + threadIdx.x) * 8;
    const float4 g0 = *reinterpret_cast<const float4*>(g + col), g1 = *reinterpret_cast<const float4*>(g + col + 4);
    gg[c][0] = g0.x; gg[c][1] = g0.y; gg[c][2] = g0.z; gg[c][3] = g0.w;
    gg[c][4] = g1.x; gg[c][5] = g1.y; gg[c][6] = g1.z; gg[c][7] = g1.w;
#pragma unroll
    for (int j = 0; j < 8; ++j) adg[c][j] = adb[c][j] = adx[c][j] = 0.f;
  }
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const float mean = mean_in[row], rstd = rstd_in[row];
    const bf16* xr = x + (long long)row * d;
    const bf16* dyr = dy + (long long)row * d;
    float xh[NCW][8], dg_[NCW][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < NCW; ++c) {
      const int col = (c * 128 + threadIdx.x) * 8;
      float xv[8], dv[8];
      unpack8(*reinterpret_cast<const uint4*>(xr + col), xv);
      unpack8(*reinterpret_cast<const uint4*>(dyr + col), dv);
      if constexpr (DIVMAX) {
#pragma unroll
        for (int j = 0; j < 8; ++j) xv[j] = __fdiv_rn(xv[j], m_in[row]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float h = (xv[j] - mean) * rstd;
        const float t = dv[j] * gg[c][j];
        xh[c][j] = h;
        dg_[c][j] = t;
        s1 += t;
        s2 += t * h;
        adg[c][j] += dv[j] * h;
        adb[c][j] += dv[j];
      }
    }
    const float2 ss = block128_sum2(s1, s2, red);
    const float c1 = ss.x * (1.f / d), c2 = ss.y * (1.f / d);
#pragma unroll
    for (int c = 0; c < NCW; ++c) {
      const int col = (c * 128 + threadIdx.x) * 8;
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (dg_[c][j] - c1 - xh[c][j] * c2) * rstd;
      if constexpr (DIVMAX) {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = __fdiv_rn(o[j], m_in[row]);
      }
      if (dres) {
        float r[8];
        unpack8(*reinterpret_cast<const uint4*>(dres + (long long)row * d + col), r);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += r[j];
      }
      ln_bwd_store8<DROP>(o, dx, dxm, row, d, col, dxsum != nullptr, dr, adx[c]);
    }
  }
#pragma unroll
  for (int c = 0; c < NCW; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = (c * 128 + threadIdx.x) * 8 + j;
      const long long o = (long long)blockIdx.x * d + col;  // this block's partial row
      dg[o] = adg[c][j];
      db[o] = adb[c][j];
      if (dxsum) dxsum[o] = adx[c][j];
    }
}

// ------------------------------------------------------------------------------------------------ LayerScale
// y = bf16(x + s[c] * o), one 16-byte vector (8 columns) per thread and grid-stride step; nv = d / 8.
__global__ void __launch_bounds__(256)
layer_scale_residual_fwd_kernel(const bf16* __restrict__ o, const bf16* __restrict__ x, const float* __restrict__ s,
                                bf16* __restrict__ y, long long total, int nv) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % nv) << 3;
    float ov[8];
    unpack8(reinterpret_cast<const uint4*>(o)[i], ov);
    ln_add_scaled_res8(x + i * 8, s + col, ov);
    reinterpret_cast<uint4*>(y)[i] = pack8(ov);
  }
}

// dv = bf16(s * dy (* keep * scale)), ds += colsum(dy * v), db += colsum(dv as stored).  grid (d / 256, row splits):
// lane -> 8 columns of the block's 256, the 8 warps stride over rows; one partial row of ds (and db) per block, summed
// in block order by reduce_rows_add.  SAND: v = (o - mean) * rstd * g + b from the stored o, the expression of
// layernorm_fwd_kernel.
template <bool SAND, bool DROP>
__global__ void __launch_bounds__(256)
layer_scale_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ v, const float* __restrict__ s,
                       const float* __restrict__ g, const float* __restrict__ b, const float* __restrict__ mean_in,
                       const float* __restrict__ rstd_in, bf16* __restrict__ dv, float* __restrict__ ds_part,
                       float* __restrict__ db_part, int rows, int d, const db200_dropout dr) {
  __shared__ float red[8][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + lane * 8;
  float ss[8], gg[8], bb[8], ads[8], adb[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    ss[j] = s[col + j];
    gg[j] = SAND ? g[col + j] : 1.f;
    bb[j] = SAND ? b[col + j] : 0.f;
    ads[j] = adb[j] = 0.f;
  }
  for (int r = blockIdx.y * 8 + warp; r < rows; r += gridDim.y * 8) {
    const long long off = (long long)r * d + col;
    float dyv[8], vv[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(dy + off), dyv);
    unpack8(*reinterpret_cast<const uint4*>(v + off), vv);
    if constexpr (SAND) {
      const float mean = mean_in[r], rstd = rstd_in[r];
#pragma unroll
      for (int j = 0; j < 8; ++j) vv[j] = (vv[j] - mean) * rstd * gg[j] + bb[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      ads[j] += dyv[j] * vv[j];
      o[j] = ss[j] * dyv[j];
    }
    if constexpr (DROP) {
      float m[8];
      dropout_mul8(dr, r, d, col, m);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] *= m[j];
    }
    const uint4 packed = pack8(o);
    *reinterpret_cast<uint4*>(dv + off) = packed;
    if (db_part) {
      unpack8(packed, o);
#pragma unroll
      for (int j = 0; j < 8; ++j) adb[j] += o[j];
    }
  }
  const int npass = db_part ? 2 : 1;
#pragma unroll 1
  for (int pass = 0; pass < npass; ++pass) {
#pragma unroll
    for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = pass == 0 ? ads[j] : adb[j];
    __syncthreads();
    const int c = threadIdx.x;
    float t = red[0][c];
#pragma unroll
    for (int w = 1; w < 8; ++w) t += red[w][c];
    (pass == 0 ? ds_part : db_part)[(long long)blockIdx.y * d + blockIdx.x * 256 + c] = t;
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ column sums
// grid: (ceil(cols/256), row_splits).  lane -> 8 columns, warps stride over rows.
__global__ void __launch_bounds__(256)
colsum_kernel(const bf16* __restrict__ x, long long ld, int rows, int cols, float* __restrict__ out) {
  __shared__ float red[8][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + lane * 8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col < cols) {  // cols % 8 == 0 is checked on the host
    for (int r = blockIdx.y * 8 + warp; r < rows; r += gridDim.y * 8) {
      float v[8];
      unpack8(*reinterpret_cast<const uint4*>(x + (long long)r * ld + col), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = acc[j];
  __syncthreads();
  const int c = threadIdx.x;
  if (blockIdx.x * 256 + c < cols) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][c];
    out[(long long)blockIdx.y * cols + blockIdx.x * 256 + c] = s;  // partial of row split blockIdx.y
  }
}

// ------------------------------------------------------------------------------------------------ casts
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, size_t n) {
  const size_t nv = n >> 3;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(src)[2 * i], b = reinterpret_cast<const float4*>(src)[2 * i + 1];
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    reinterpret_cast<uint4*>(dst)[i] = pack8(f);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 7)) dst[(nv << 3) + threadIdx.x] = __float2bfloat16(src[(nv << 3) + threadIdx.x]);
}
__global__ void cast_bf16_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst, size_t n) {
  const size_t nv = n >> 3;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
    float f[8];
    unpack8(reinterpret_cast<const uint4*>(src)[i], f);
    reinterpret_cast<float4*>(dst)[2 * i] = make_float4(f[0], f[1], f[2], f[3]);
    reinterpret_cast<float4*>(dst)[2 * i + 1] = make_float4(f[4], f[5], f[6], f[7]);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 7)) dst[(nv << 3) + threadIdx.x] = __bfloat162float(src[(nv << 3) + threadIdx.x]);
}

// x (f32) -> hi = bf16(x), lo = bf16(x - hi): x = hi + lo up to 2^-16 relative.  Lets an fp32 operand go through the
// bf16 tensor pipe as two products with fp32 accumulation (used for the VAE codebook matmuls, which the reference
// keeps in fp32: src/vae_tf/models.py:115-118).
__global__ void split_f32_kernel(const float* __restrict__ src, bf16* __restrict__ hi, bf16* __restrict__ lo, size_t n) {
  const size_t nv = n >> 3;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(src)[2 * i], b = reinterpret_cast<const float4*>(src)[2 * i + 1];
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    float h[8], l[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      h[j] = __bfloat162float(__float2bfloat16(f[j]));
      l[j] = f[j] - h[j];
    }
    reinterpret_cast<uint4*>(hi)[i] = pack8(h);
    if (lo) reinterpret_cast<uint4*>(lo)[i] = pack8(l);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 7)) {
    const size_t i = (nv << 3) + threadIdx.x;
    const bf16 hh = __float2bfloat16(src[i]);
    hi[i] = hh;
    if (lo) lo[i] = __float2bfloat16(src[i] - __bfloat162float(hh));
  }
}

// ------------------------------------------------------------------------------------------------ CE finish
// Combine the per-vocab-tile (max, sum-exp) partials into lse, loss_row; block-sum the loss.
// Partials are stored [n_tiles][M] (tile-major): the GEMM epilogue's 32 lanes = 32 consecutive rows write one 128-byte
// line per store.  Here a block owns 32 consecutive rows; warp g of 8 folds tiles g, g+8, ... (every load is one
// 128-byte line), then the 8 partial (max, sum) pairs of a row are merged through shared memory.
constexpr int CEF_ROWS = 32, CEF_GROUPS = 8;
// warp g folds tiles g, g + 8, ... of row `row` into one (max, sum) pair, stored at sm_m / sm_s[g][r]; block barrier
__device__ __forceinline__ void ce_fold_tiles(const float* __restrict__ part_max, const float* __restrict__ part_sum,
                                              int M, int n_tiles, int row, int r, int g,
                                              float (*sm_m)[CEF_ROWS], float (*sm_s)[CEF_ROWS]) {
  float m = -INFINITY, s = 0.f;
  if (row < M) {
    constexpr int U = 4;  // tiles in flight per thread: the loop is load-latency bound otherwise
    for (int t0 = g; t0 < n_tiles; t0 += CEF_GROUPS * U) {
      float pm[U], ps[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int t = t0 + u * CEF_GROUPS;
        pm[u] = t < n_tiles ? __ldg(part_max + (long long)t * M + row) : -INFINITY;
        ps[u] = t < n_tiles ? __ldg(part_sum + (long long)t * M + row) : 0.f;
      }
      float mn = m;
#pragma unroll
      for (int u = 0; u < U; ++u) mn = fmaxf(mn, pm[u]);
      if (mn > -INFINITY) {
        s *= expf(m - mn);  // expf(-inf) = 0 on the first valid tile
#pragma unroll
        for (int u = 0; u < U; ++u) s += ps[u] * expf(pm[u] - mn);  // tiles with no valid column: 0 * exp(-inf) = 0
        m = mn;
      }
    }
  }
  sm_m[g][r] = m;
  sm_s[g][r] = s;
  __syncthreads();
}
// lse of row r of the block from the CEF_GROUPS folded pairs
__device__ __forceinline__ float ce_merge_lse(float (*sm_m)[CEF_ROWS], float (*sm_s)[CEF_ROWS], int r) {
  float mm = -INFINITY;
#pragma unroll
  for (int i = 0; i < CEF_GROUPS; ++i) mm = fmaxf(mm, sm_m[i][r]);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < CEF_GROUPS; ++i)
    if (sm_m[i][r] > -INFINITY) ss += sm_s[i][r] * expf(sm_m[i][r] - mm);
  return mm + logf(ss);
}

__global__ void __launch_bounds__(CEF_ROWS * CEF_GROUPS)
ce_finish_kernel(const float* __restrict__ part_max, const float* __restrict__ part_sum,
                 const float* __restrict__ label_logit, float* __restrict__ lse, float* __restrict__ loss_rows,
                 float* __restrict__ loss_sum, int M, int n_tiles) {
  __shared__ float sm_m[CEF_GROUPS][CEF_ROWS], sm_s[CEF_GROUPS][CEF_ROWS];
  const int r = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int row = blockIdx.x * CEF_ROWS + r;
  ce_fold_tiles(part_max, part_sum, M, n_tiles, row, r, g, sm_m, sm_s);
  if (g == 0) {
    float loss = 0.f;
    if (row < M) {
      const float l = ce_merge_lse(sm_m, sm_s, r);
      loss = l - label_logit[row];
      lse[row] = l;
      loss_rows[row] = loss;
    }
    loss = warp_sum(loss);
    if (r == 0) loss_sum[blockIdx.x] = loss;  // per-block partial, summed in block order by the launcher
  }
}

// Weighted finish: loss_rows = CE + z lse^2; per-block partials [blocks][4] of (sum a loss_rows, text CE, image CE,
// z lse^2), added in block order by the launcher.
__global__ void __launch_bounds__(CEF_ROWS * CEF_GROUPS)
ce_finish_weighted_kernel(const float* __restrict__ part_max, const float* __restrict__ part_sum,
                          const float* __restrict__ label_logit, float* __restrict__ lse, float* __restrict__ loss_rows,
                          float* __restrict__ partials, int M, int n_tiles, const db200_ce_weights w) {
  __shared__ float sm_m[CEF_GROUPS][CEF_ROWS], sm_s[CEF_GROUPS][CEF_ROWS];
  const int r = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int row = blockIdx.x * CEF_ROWS + r;
  ce_fold_tiles(part_max, part_sum, M, n_tiles, row, r, g, sm_m, sm_s);
  if (g == 0) {
    float weighted = 0.f, ce_text = 0.f, ce_image = 0.f, zterm = 0.f;
    if (row < M) {
      const float l = ce_merge_lse(sm_m, sm_s, r);
      const float ce = l - label_logit[row];
      zterm = w.z_loss * l * l;
      const float loss = ce + zterm;
      const bool text = (row % w.period) < w.text_rows;
      weighted = (text ? w.a_text : w.a_image) * loss;
      (text ? ce_text : ce_image) = ce;
      lse[row] = l;
      loss_rows[row] = loss;
    }
    weighted = warp_sum(weighted);
    ce_text = warp_sum(ce_text);
    ce_image = warp_sum(ce_image);
    zterm = warp_sum(zterm);
    if (r == 0) {
      float* o = partials + 4 * (long long)blockIdx.x;
      o[0] = weighted; o[1] = ce_text; o[2] = ce_image; o[3] = zterm;
    }
  }
}

}  // namespace db200

using namespace db200;

extern "C" int db200_embed_fwd(db200_stream_t stream_, const int32_t* ids, const void* wte, const void* wpe,
                               void* out, int B, int S, int d, int V) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && S > 0 && d > 0 && V > 0 && d % 8 == 0, DB200_E_INVALID,
                "embed_fwd: need B,S,V > 0 and d %% 8 == 0 (got B=%d S=%d d=%d V=%d)", B, S, d, V);
  DB200_REQUIRE(ids && aligned16(wte) && aligned16(wpe) && aligned16(out), DB200_E_ALIGN,
                "embed_fwd: NULL or unaligned pointer");
  const long long total = (long long)B * S * (d / 8);
  const int blocks = (int)((total + 255) / 256 < sm_count() * 16 ? (total + 255) / 256 : sm_count() * 16);
  embed_fwd_kernel<<<blocks, 256, 0, stream>>>(ids, (const bf16*)wte, (const bf16*)wpe, (bf16*)out, B * S, S, d, V);
  return check_launch("embed_fwd_kernel");
}

extern "C" int db200_embed_fwd_ex(db200_stream_t stream_, const int32_t* ids, const void* wte, const void* wpe,
                                  void* out, int B, int S, int d, int V, const db200_dropout* wte_drop,
                                  const db200_dropout* wpe_drop) {
  if (!dropout_active(wte_drop) && !dropout_active(wpe_drop))
    return db200_embed_fwd(stream_, ids, wte, wpe, out, B, S, d, V);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && S > 0 && d > 0 && V > 0 && d % 8 == 0, DB200_E_INVALID,
                "embed_fwd: need B,S,V > 0 and d %% 8 == 0 (got B=%d S=%d d=%d V=%d)", B, S, d, V);
  DB200_REQUIRE(ids && aligned16(wte) && aligned16(wpe) && aligned16(out), DB200_E_ALIGN,
                "embed_fwd: NULL or unaligned pointer");
  db200_dropout keep_all{};  // threshold 0: every element kept, scale 1
  keep_all.scale = 1.f;
  const long long total = (long long)B * S * (d / 8);
  const int blocks = (int)((total + 255) / 256 < sm_count() * 16 ? (total + 255) / 256 : sm_count() * 16);
  embed_fwd_drop_kernel<<<blocks, 256, 0, stream>>>(ids, (const bf16*)wte, (const bf16*)wpe, (bf16*)out, B * S, S, d,
                                                    V, dropout_active(wte_drop) ? *wte_drop : keep_all,
                                                    dropout_active(wpe_drop) ? *wpe_drop : keep_all);
  return check_launch("embed_fwd_drop_kernel");
}

extern "C" int64_t db200_embed_bwd_workspace_bytes(int d, int V) {
  return (int64_t)V * d * (int64_t)sizeof(unsigned long long);
}

extern "C" int db200_embed_bwd(db200_stream_t stream_, const int32_t* ids, const void* dx, float* dwte, float* dwpe,
                               int B, int S, int d, int V, void* workspace, int64_t workspace_bytes) {
  return db200_embed_bwd_ex(stream_, ids, dx, dwte, dwpe, B, S, d, V, workspace, workspace_bytes, nullptr, nullptr);
}

// SCALE: every dx element times alpha before it is summed (db200_embed_bwd_scaled)
template <bool SCALE>
static int embed_bwd_impl(cudaStream_t stream, const int32_t* ids, const void* dx, float* dwte, float* dwpe, int B,
                          int S, int d, int V, void* workspace, int64_t workspace_bytes, const db200_dropout* wte_drop,
                          const db200_dropout* wpe_drop, float alpha) {
  const db200_dropout* dw = dropout_active(wte_drop) ? wte_drop : nullptr;
  const db200_dropout* dp = dropout_active(wpe_drop) ? wpe_drop : nullptr;
  DB200_REQUIRE(B > 0 && S > 0 && d > 0 && V > 0 && d % 8 == 0, DB200_E_INVALID,
                "embed_bwd: need B,S,V > 0 and d %% 8 == 0");
  DB200_REQUIRE(ids && aligned16(dx) && dwte && dwpe, DB200_E_ALIGN, "embed_bwd: NULL or unaligned pointer");
  const long long total = (long long)(((long long)B * S + EMB_STRIP - 1) / EMB_STRIP) * (d / 8);
  const int blocks = (int)((total + 255) / 256 < sm_count() * 16 ? (total + 255) / 256 : sm_count() * 16);
  const long long n_wte = (long long)V * d;
  DB200_REQUIRE(workspace_ok(workspace, workspace_bytes, db200_embed_bwd_workspace_bytes(d, V)), DB200_E_INVALID,
                "embed_bwd: needs an aligned workspace of db200_embed_bwd_workspace_bytes() bytes");
  auto* acc64 = static_cast<unsigned long long*>(workspace);
  DB200_CUDA(cudaMemsetAsync(acc64, 0, (size_t)n_wte * sizeof(unsigned long long), stream));
  if (dw) embed_bwd_wte_kernel<true, SCALE><<<blocks, 256, 0, stream>>>(ids, (const bf16*)dx, acc64, B * S, d, V, *dw, alpha);
  else    embed_bwd_wte_kernel<false, SCALE><<<blocks, 256, 0, stream>>>(ids, (const bf16*)dx, acc64, B * S, d, V, db200_dropout{}, alpha);
  int rc = check_launch("embed_bwd_wte_kernel");
  if (rc != DB200_OK) return rc;
  const long long fblocks = (n_wte + 255) / 256 < sm_count() * 16 ? (n_wte + 255) / 256 : sm_count() * 16;
  embed_fixed_flush_kernel<<<(int)fblocks, 256, 0, stream>>>(acc64, dwte, n_wte);
  rc = check_launch("embed_fixed_flush_kernel");
  if (rc != DB200_OK) return rc;
  const int total_pe = S * (d / 8);
  if (dp) embed_bwd_wpe_kernel<true, SCALE><<<(total_pe + 127) / 128, 128, 0, stream>>>((const bf16*)dx, dwpe, B, S, d, *dp, alpha);
  else    embed_bwd_wpe_kernel<false, SCALE><<<(total_pe + 127) / 128, 128, 0, stream>>>((const bf16*)dx, dwpe, B, S, d, db200_dropout{}, alpha);
  return check_launch("embed_bwd_wpe_kernel");
}

extern "C" int db200_embed_bwd_ex(db200_stream_t stream_, const int32_t* ids, const void* dx, float* dwte,
                                  float* dwpe, int B, int S, int d, int V, void* workspace, int64_t workspace_bytes,
                                  const db200_dropout* wte_drop, const db200_dropout* wpe_drop) {
  return embed_bwd_impl<false>(reinterpret_cast<cudaStream_t>(stream_), ids, dx, dwte, dwpe, B, S, d, V, workspace,
                               workspace_bytes, wte_drop, wpe_drop, 1.f);
}

extern "C" int db200_embed_bwd_scaled(db200_stream_t stream_, const int32_t* ids, const void* dx, float* dwte,
                                      float* dwpe, int B, int S, int d, int V, void* workspace, int64_t workspace_bytes,
                                      const db200_dropout* wte_drop, const db200_dropout* wpe_drop, float alpha) {
  return embed_bwd_impl<true>(reinterpret_cast<cudaStream_t>(stream_), ids, dx, dwte, dwpe, B, S, d, V, workspace,
                              workspace_bytes, wte_drop, wpe_drop, alpha);
}

extern "C" int db200_shift_labels(db200_stream_t stream_, const int32_t* ids, int32_t* labels, int B, int S,
                                  int eos_id) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && S > 0 && ids && labels, DB200_E_INVALID, "shift_labels: bad arguments");
  shift_labels_kernel<<<(B * S + 255) / 256, 256, 0, stream>>>(ids, labels, B, S, eos_id);
  return check_launch("shift_labels_kernel");
}

extern "C" int db200_assemble_tokens(db200_stream_t stream_, const int32_t* text_ids, const int32_t* image_idx,
                                     int32_t* tokens, int B, int text_len, int image_len, int image_offset) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && text_len >= 0 && image_len >= 0 && text_len + image_len > 0 && tokens &&
                    (text_len == 0 || text_ids) && (image_len == 0 || image_idx),
                DB200_E_INVALID, "assemble_tokens: bad arguments");
  const int n = B * (text_len + image_len);
  assemble_tokens_kernel<<<(n + 255) / 256, 256, 0, stream>>>(text_ids, image_idx, tokens, B, text_len, image_len,
                                                            image_offset);
  return check_launch("assemble_tokens_kernel");
}

extern "C" int db200_assemble_tokens_ex(db200_stream_t stream_, const int32_t* text_ids, const int32_t* image_idx,
                                        int32_t* tokens, int B, int text_len, int image_len, int image_offset,
                                        int32_t pad_id, const db200_dropout* caption_drop) {
  if (!dropout_active(caption_drop))
    return db200_assemble_tokens(stream_, text_ids, image_idx, tokens, B, text_len, image_len, image_offset);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && text_len >= 0 && image_len >= 0 && text_len + image_len > 0 && tokens &&
                    (text_len == 0 || text_ids) && (image_len == 0 || image_idx),
                DB200_E_INVALID, "assemble_tokens_ex: bad arguments");
  DB200_REQUIRE(pad_id >= 0 && caption_drop->row0 >= 0, DB200_E_INVALID, "assemble_tokens_ex: pad_id %d row0 %lld",
                pad_id, (long long)caption_drop->row0);
  const int n = B * (text_len + image_len);
  assemble_tokens_drop_kernel<<<(n + 255) / 256, 256, 0, stream>>>(text_ids, image_idx, tokens, B, text_len, image_len,
                                                                  image_offset, pad_id, *caption_drop);
  return check_launch("assemble_tokens_drop_kernel");
}

extern "C" int db200_assemble_tokens_pp(db200_stream_t stream_, const int32_t* text_ids, const int32_t* image_idx,
                                        int32_t* tokens, int B, int text_len, int image_len, int image_offset,
                                        int32_t pad_id, int32_t pad_base, const db200_dropout* caption_drop) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && text_len >= 0 && image_len >= 0 && text_len + image_len > 0 && tokens &&
                    (text_len == 0 || text_ids) && (image_len == 0 || image_idx),
                DB200_E_INVALID, "assemble_tokens_pp: bad arguments");
  DB200_REQUIRE(pad_id >= 0 && pad_base >= 0 && (long long)pad_base + text_len <= 2147483647LL, DB200_E_INVALID,
                "assemble_tokens_pp: pad_id %d pad_base %d", pad_id, pad_base);
  const bool drop = dropout_active(caption_drop);
  DB200_REQUIRE(!drop || caption_drop->row0 >= 0, DB200_E_INVALID, "assemble_tokens_pp: row0 %lld",
                (long long)caption_drop->row0);
  const int n = B * (text_len + image_len);
  if (drop) {
    assemble_tokens_pp_kernel<true><<<(n + 255) / 256, 256, 0, stream>>>(text_ids, image_idx, tokens, B, text_len,
                                                                         image_len, image_offset, pad_id, pad_base,
                                                                         *caption_drop);
  } else {
    assemble_tokens_pp_kernel<false><<<(n + 255) / 256, 256, 0, stream>>>(text_ids, image_idx, tokens, B, text_len,
                                                                          image_len, image_offset, pad_id, pad_base,
                                                                          db200_dropout{});
  }
  return check_launch("assemble_tokens_pp_kernel");
}

extern "C" int db200_pos_compose(db200_stream_t stream_, const void* wpe, const void* image_row, const void* image_col,
                                 void* pos, int text_len, int grid_w, int d) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(text_len >= 0 && grid_w > 0 && d > 0 && d % 8 == 0, DB200_E_INVALID,
                "pos_compose: need text_len >= 0, grid_w > 0 and d %% 8 == 0 (got %d %d %d)", text_len, grid_w, d);
  DB200_REQUIRE((text_len == 0 || aligned16(wpe)) && aligned16(image_row) && aligned16(image_col) && aligned16(pos),
                DB200_E_ALIGN, "pos_compose: NULL or unaligned pointer");
  const long long total = ((long long)text_len + (long long)grid_w * grid_w) * (d / 8);
  const int blocks = (int)((total + 255) / 256 < sm_count() * 16 ? (total + 255) / 256 : sm_count() * 16);
  pos_compose_kernel<<<blocks, 256, 0, stream>>>((const bf16*)wpe, (const bf16*)image_row, (const bf16*)image_col,
                                                 (bf16*)pos, text_len, grid_w, d);
  return check_launch("pos_compose_kernel");
}

extern "C" int db200_pos_fold(db200_stream_t stream_, const float* dpos, float* dwpe, float* dimage_row,
                              float* dimage_col, int text_len, int grid_w, int d) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(text_len >= 0 && grid_w > 0 && d > 0 && d % 8 == 0, DB200_E_INVALID,
                "pos_fold: need text_len >= 0, grid_w > 0 and d %% 8 == 0 (got %d %d %d)", text_len, grid_w, d);
  DB200_REQUIRE(aligned16(dpos) && (text_len == 0 || aligned16(dwpe)) && aligned16(dimage_row) &&
                    aligned16(dimage_col),
                DB200_E_ALIGN, "pos_fold: NULL or unaligned pointer");
  const long long total = ((long long)text_len + 2LL * grid_w) * (d / 8);
  const int blocks = (int)((total + 255) / 256 < sm_count() * 16 ? (total + 255) / 256 : sm_count() * 16);
  pos_fold_kernel<<<blocks, 256, 0, stream>>>(dpos, dwpe, dimage_row, dimage_col, text_len, grid_w, d);
  return check_launch("pos_fold_kernel");
}

extern "C" int db200_layernorm_fwd(db200_stream_t stream_, const void* x, const float* g, const float* b, void* y,
                                   float* mean, float* rstd, int rows, int d, float eps) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(rows > 0, DB200_E_INVALID, "layernorm_fwd: rows must be positive");
  DB200_REQUIRE(aligned16(x) && aligned16(y) && aligned16(g) && aligned16(b) && mean && rstd, DB200_E_ALIGN,
                "layernorm_fwd: NULL or unaligned pointer");
  const int grid = (rows + 3) / 4;
  const bf16* xp = (const bf16*)x;
  bf16* yp = (bf16*)y;
  switch (d) {
    case 256:  layernorm_fwd_kernel<1><<<grid, 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps); break;
    case 512:  layernorm_fwd_kernel<2><<<grid, 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps); break;
    case 768:  layernorm_fwd_kernel<3><<<grid, 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps); break;
    case 1024: layernorm_fwd_kernel<4><<<grid, 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps); break;
    case 2048: layernorm_fwd_kernel<8><<<grid, 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps); break;
    case 4096: layernorm_fwd_wide_kernel<4><<<min(rows, sm_count() * 16), 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps); break;
    default:
      return set_error(DB200_E_UNSUPPORTED, "layernorm: d=%d not in {256,512,768,1024,2048,4096}", d);
  }
  return check_launch("layernorm_fwd_kernel");
}

extern "C" int db200_layernorm_residual_fwd(db200_stream_t stream_, const void* o, const void* x_res, const float* g,
                                            const float* b, void* y, float* mean, float* rstd, int rows, int d,
                                            float eps) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(rows > 0, DB200_E_INVALID, "layernorm_residual_fwd: rows must be positive");
  DB200_REQUIRE(o && x_res && y && g && b && mean && rstd, DB200_E_INVALID, "layernorm_residual_fwd: NULL pointer");
  DB200_REQUIRE(aligned16(o) && aligned16(x_res) && aligned16(y) && aligned16(g) && aligned16(b), DB200_E_ALIGN,
                "layernorm_residual_fwd: unaligned pointer");
  const int grid = (rows + 3) / 4;
  const bf16* op = (const bf16*)o;
  const bf16* rp = (const bf16*)x_res;
  bf16* yp = (bf16*)y;
  switch (d) {
    case 256:  layernorm_fwd_kernel<1, true><<<grid, 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp); break;
    case 512:  layernorm_fwd_kernel<2, true><<<grid, 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp); break;
    case 768:  layernorm_fwd_kernel<3, true><<<grid, 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp); break;
    case 1024: layernorm_fwd_kernel<4, true><<<grid, 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp); break;
    case 2048: layernorm_fwd_kernel<8, true><<<grid, 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp); break;
    case 4096: layernorm_fwd_wide_kernel<4, true><<<min(rows, sm_count() * 16), 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp); break;
    default:
      return set_error(DB200_E_UNSUPPORTED, "layernorm_residual_fwd: d=%d not in {256,512,768,1024,2048,4096}", d);
  }
  return check_launch("layernorm_residual_fwd_kernel");
}

extern "C" int db200_layernorm_scale_residual_fwd(db200_stream_t stream_, const void* o, const void* x_res,
                                                  const float* g, const float* b, const float* s, void* y, float* mean,
                                                  float* rstd, int rows, int d, float eps) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(rows > 0, DB200_E_INVALID, "layernorm_scale_residual_fwd: rows must be positive");
  DB200_REQUIRE(o && x_res && y && g && b && s && mean && rstd, DB200_E_INVALID,
                "layernorm_scale_residual_fwd: NULL pointer");
  DB200_REQUIRE(aligned16(o) && aligned16(x_res) && aligned16(y) && aligned16(g) && aligned16(b) && aligned16(s),
                DB200_E_ALIGN, "layernorm_scale_residual_fwd: unaligned pointer");
  const int grid = (rows + 3) / 4;
  const bf16* op = (const bf16*)o;
  const bf16* rp = (const bf16*)x_res;
  bf16* yp = (bf16*)y;
  switch (d) {
    case 256:  layernorm_fwd_kernel<1, true, true><<<grid, 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp, s); break;
    case 512:  layernorm_fwd_kernel<2, true, true><<<grid, 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp, s); break;
    case 768:  layernorm_fwd_kernel<3, true, true><<<grid, 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp, s); break;
    case 1024: layernorm_fwd_kernel<4, true, true><<<grid, 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp, s); break;
    case 2048: layernorm_fwd_kernel<8, true, true><<<grid, 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp, s); break;
    case 4096: layernorm_fwd_wide_kernel<4, true, true><<<min(rows, sm_count() * 16), 128, 0, stream>>>(op, g, b, yp, mean, rstd, rows, eps, rp, s); break;
    default:
      return set_error(DB200_E_UNSUPPORTED, "layernorm_scale_residual_fwd: d=%d not in {256,512,768,1024,2048,4096}",
                       d);
  }
  return check_launch("layernorm_scale_residual_fwd_kernel");
}

extern "C" int db200_layernorm_divmax_fwd(db200_stream_t stream_, const void* x, const float* g, const float* b,
                                          void* y, float* mean, float* rstd, float* m, int rows, int d, float eps) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(rows > 0, DB200_E_INVALID, "layernorm_divmax_fwd: rows must be positive");
  DB200_REQUIRE(x && y && g && b && mean && rstd && m, DB200_E_INVALID, "layernorm_divmax_fwd: NULL pointer");
  DB200_REQUIRE(aligned16(x) && aligned16(y) && aligned16(g) && aligned16(b), DB200_E_ALIGN,
                "layernorm_divmax_fwd: unaligned pointer");
  const int grid = (rows + 3) / 4;
  const bf16* xp = (const bf16*)x;
  bf16* yp = (bf16*)y;
  switch (d) {
    case 256:  layernorm_fwd_kernel<1, false, false, true><<<grid, 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps, nullptr, nullptr, m); break;
    case 512:  layernorm_fwd_kernel<2, false, false, true><<<grid, 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps, nullptr, nullptr, m); break;
    case 768:  layernorm_fwd_kernel<3, false, false, true><<<grid, 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps, nullptr, nullptr, m); break;
    case 1024: layernorm_fwd_kernel<4, false, false, true><<<grid, 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps, nullptr, nullptr, m); break;
    case 2048: layernorm_fwd_kernel<8, false, false, true><<<grid, 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps, nullptr, nullptr, m); break;
    case 4096: layernorm_fwd_wide_kernel<4, false, false, true><<<min(rows, sm_count() * 16), 128, 0, stream>>>(xp, g, b, yp, mean, rstd, rows, eps, nullptr, nullptr, m); break;
    default:
      return set_error(DB200_E_UNSUPPORTED, "layernorm_divmax_fwd: d=%d not in {256,512,768,1024,2048,4096}", d);
  }
  return check_launch("layernorm_divmax_fwd_kernel");
}

extern "C" int db200_layer_scale_residual_fwd(db200_stream_t stream_, const void* o, const void* x_res, const float* s,
                                              void* y, int rows, int d) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(rows > 0 && d > 0 && d % 8 == 0, DB200_E_INVALID,
                "layer_scale_residual_fwd: need rows > 0 and d a positive multiple of 8 (got rows=%d d=%d)", rows, d);
  DB200_REQUIRE(o && x_res && s && y, DB200_E_INVALID, "layer_scale_residual_fwd: NULL pointer");
  DB200_REQUIRE(aligned16(o) && aligned16(x_res) && aligned16(s) && aligned16(y), DB200_E_ALIGN,
                "layer_scale_residual_fwd: unaligned pointer");
  const long long total = (long long)rows * (d / 8);
  const long long want = (total + 255) / 256;
  const int grid = (int)(want < (long long)sm_count() * 16 ? want : (long long)sm_count() * 16);
  layer_scale_residual_fwd_kernel<<<grid, 256, 0, stream>>>((const bf16*)o, (const bf16*)x_res, s, (bf16*)y, total,
                                                            d / 8);
  return check_launch("layer_scale_residual_fwd_kernel");
}

static int layer_scale_bwd_splits(int rows, int d) {
  const int gx = d / 256;
  int gy = (sm_count() * 4 + gx - 1) / gx;
  if (gy > (rows + 7) / 8) gy = (rows + 7) / 8;
  return gy < 1 ? 1 : gy;
}

extern "C" int64_t db200_layer_scale_bwd_workspace_bytes(int rows, int d) {
  if (rows <= 0 || d <= 0 || d % 256) return 0;
  return (int64_t)2 * layer_scale_bwd_splits(rows, d) * d * (int64_t)sizeof(float);
}

extern "C" int db200_layer_scale_bwd(db200_stream_t stream_, const void* dy, const void* v, const float* s,
                                     const float* g, const float* b, const float* mean, const float* rstd, void* dv,
                                     float* ds, float* db, const db200_dropout* drop, int rows, int d, void* workspace,
                                     int64_t workspace_bytes) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(rows > 0 && d > 0 && d % 256 == 0, DB200_E_INVALID,
                "layer_scale_bwd: need rows > 0 and d a positive multiple of 256 (got rows=%d d=%d)", rows, d);
  DB200_REQUIRE(dy && v && s && dv && ds, DB200_E_INVALID, "layer_scale_bwd: NULL pointer");
  DB200_REQUIRE(aligned16(dy) && aligned16(v) && aligned16(dv), DB200_E_ALIGN, "layer_scale_bwd: unaligned pointer");
  const bool sand = g != nullptr;
  DB200_REQUIRE(!sand || (b && mean && rstd), DB200_E_INVALID,
                "layer_scale_bwd: the sandwich form (g given) needs b, mean and rstd");
  DB200_REQUIRE(!(sand && dropout_active(drop)), DB200_E_INVALID,
                "layer_scale_bwd: the sandwich form takes no dropout (the LayerNorm backward applies it)");
  const int gy = layer_scale_bwd_splits(rows, d);
  DB200_REQUIRE(workspace_ok(workspace, workspace_bytes, db200_layer_scale_bwd_workspace_bytes(rows, d)),
                DB200_E_INVALID, "layer_scale_bwd: needs an aligned workspace of db200_layer_scale_bwd_workspace_bytes() bytes");
  float* ds_part = static_cast<float*>(workspace);
  float* db_part = db ? ds_part + (size_t)gy * d : nullptr;
  const dim3 grid(d / 256, gy);
  const bf16 *dyp = (const bf16*)dy, *vp = (const bf16*)v;
  bf16* dvp = (bf16*)dv;
  if (sand)
    layer_scale_bwd_kernel<true, false><<<grid, 256, 0, stream>>>(dyp, vp, s, g, b, mean, rstd, dvp, ds_part, db_part,
                                                                  rows, d, db200_dropout{});
  else if (dropout_active(drop))
    layer_scale_bwd_kernel<false, true><<<grid, 256, 0, stream>>>(dyp, vp, s, g, b, mean, rstd, dvp, ds_part, db_part,
                                                                  rows, d, *drop);
  else
    layer_scale_bwd_kernel<false, false><<<grid, 256, 0, stream>>>(dyp, vp, s, g, b, mean, rstd, dvp, ds_part, db_part,
                                                                   rows, d, db200_dropout{});
  int rc = check_launch("layer_scale_bwd_kernel");
  if (rc == DB200_OK) rc = reduce_rows_add(stream, ds_part, gy, d, ds);
  if (rc == DB200_OK && db) rc = reduce_rows_add(stream, db_part, gy, d, db);
  return rc;
}

static int layernorm_bwd_grid(int rows, int d) {
  int grid = d == 4096 ? rows : (rows + 3) / 4;
  if (grid > sm_count() * 4) grid = sm_count() * 4;
  return grid < 1 ? 1 : grid;
}

extern "C" int64_t db200_layernorm_bwd_workspace_bytes(int rows, int d) {
  return (int64_t)3 * layernorm_bwd_grid(rows, d) * d * (int64_t)sizeof(float);
}

// the DivideMax LayerNorm backward's launch (layernorm_bwd_impl<DROP, true>); its d = 2048 rows run on the
// one-CTA-per-row kernel, which keeps the row in registers without spilling
template <bool DROP>
static int layernorm_divmax_bwd_launch(cudaStream_t stream, int grid, int d, const bf16* dyp, const bf16* xp,
                                       const float* g, const float* mean, const float* rstd, const bf16* drp, bf16* dxp,
                                       float* dg, float* db, float* dxsum, int rows, bf16* dxmp,
                                       const db200_dropout& dr, const float* m) {
  switch (d) {
    case 256:  layernorm_bwd_kernel<1, DROP, true><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr, m); break;
    case 512:  layernorm_bwd_kernel<2, DROP, true><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr, m); break;
    case 768:  layernorm_bwd_kernel<3, DROP, true><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr, m); break;
    case 1024: layernorm_bwd_kernel<4, DROP, true><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr, m); break;
    case 2048: layernorm_bwd_wide_kernel<2, DROP, true><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr, m); break;
    case 4096: layernorm_bwd_wide_kernel<4, DROP, true><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr, m); break;
    default:
      return set_error(DB200_E_UNSUPPORTED, "layernorm: d=%d not in {256,512,768,1024,2048,4096}", d);
  }
  return DB200_OK;
}

// DIVMAX: the DivideMax LayerNorm's backward (m: the rows' maxima, layernorm_divmax_bwd_launch).
template <bool DROP, bool DIVMAX = false>
static int layernorm_bwd_impl(cudaStream_t stream, const void* dy, const void* x, const float* g, const float* mean,
                              const float* rstd, const void* dres, void* dx, float* dg, float* db, float* dxsum,
                              int rows, int d, void* workspace, int64_t workspace_bytes, void* dxm,
                              const db200_dropout& dr, const float* m = nullptr) {
  DB200_REQUIRE(rows > 0, DB200_E_INVALID, "layernorm_bwd: rows must be positive");
  DB200_REQUIRE(aligned16(dy) && aligned16(x) && aligned16(dx) && aligned16(g) && mean && rstd && dg && db &&
                    aligned16(dres),
                DB200_E_ALIGN, "layernorm_bwd: NULL or unaligned pointer");
  const int grid = layernorm_bwd_grid(rows, d);
  DB200_REQUIRE(workspace_ok(workspace, workspace_bytes, db200_layernorm_bwd_workspace_bytes(rows, d)),
                DB200_E_INVALID, "layernorm_bwd: needs an aligned workspace of db200_layernorm_bwd_workspace_bytes() bytes");
  const bf16 *dyp = (const bf16*)dy, *xp = (const bf16*)x, *drp = (const bf16*)dres;
  bf16 *dxp = (bf16*)dx, *dxmp = (bf16*)dxm;
  // per-block partial rows of dg | db | dxsum, reduced in block order below
  float* ws = static_cast<float*>(workspace);
  float* const dg_out = dg;
  float* const db_out = db;
  float* const dxsum_out = dxsum;
  dg = ws;
  db = ws + (size_t)grid * d;
  dxsum = dxsum_out ? ws + (size_t)2 * grid * d : nullptr;
  if constexpr (DIVMAX) {
    const int rc0 = layernorm_divmax_bwd_launch<DROP>(stream, grid, d, dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum,
                                                      rows, dxmp, dr, m);
    if (rc0 != DB200_OK) return rc0;
  } else {
    switch (d) {
      case 256:  layernorm_bwd_kernel<1, DROP><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr); break;
      case 512:  layernorm_bwd_kernel<2, DROP><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr); break;
      case 768:  layernorm_bwd_kernel<3, DROP><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr); break;
      case 1024: layernorm_bwd_kernel<4, DROP><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr); break;
      case 2048: layernorm_bwd_kernel<8, DROP><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr); break;
      case 4096: layernorm_bwd_wide_kernel<4, DROP><<<grid, 128, 0, stream>>>(dyp, xp, g, mean, rstd, drp, dxp, dg, db, dxsum, rows, dxmp, dr); break;
      default:
        return set_error(DB200_E_UNSUPPORTED, "layernorm: d=%d not in {256,512,768,1024,2048,4096}", d);
    }
  }
  int rc = check_launch("layernorm_bwd_kernel");
  if (rc == DB200_OK) rc = reduce_rows_add(stream, dg, grid, d, dg_out);
  if (rc == DB200_OK) rc = reduce_rows_add(stream, db, grid, d, db_out);
  if (rc == DB200_OK && dxsum_out) rc = reduce_rows_add(stream, dxsum, grid, d, dxsum_out);
  return rc;
}

extern "C" int db200_layernorm_bwd_ex(db200_stream_t stream_, const void* dy, const void* x, const float* g,
                                      const float* mean, const float* rstd, const void* dres, void* dx, float* dg,
                                      float* db, float* dxsum, int rows, int d, void* workspace,
                                      int64_t workspace_bytes) {
  return layernorm_bwd_impl<false>(reinterpret_cast<cudaStream_t>(stream_), dy, x, g, mean, rstd, dres, dx, dg, db,
                                   dxsum, rows, d, workspace, workspace_bytes, nullptr, db200_dropout{});
}

extern "C" int db200_layernorm_bwd_dropout(db200_stream_t stream_, const void* dy, const void* x, const float* g,
                                           const float* mean, const float* rstd, const void* dres, void* dx,
                                           void* dxm, float* dg, float* db, float* dxsum, int rows, int d,
                                           const db200_dropout* drop, void* workspace, int64_t workspace_bytes) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(aligned16(dxm) && dxm, DB200_E_ALIGN, "layernorm_bwd_dropout: NULL or unaligned dxm");
  if (!dropout_active(drop)) {  // keep everything: dxm = dx
    const int rc = layernorm_bwd_impl<false>(stream, dy, x, g, mean, rstd, dres, dx, dg, db, dxsum, rows, d, workspace,
                                             workspace_bytes, nullptr, db200_dropout{});
    if (rc != DB200_OK) return rc;
    DB200_CUDA(cudaMemcpyAsync(dxm, dx, (size_t)rows * d * sizeof(bf16), cudaMemcpyDeviceToDevice, stream));
    return DB200_OK;
  }
  return layernorm_bwd_impl<true>(stream, dy, x, g, mean, rstd, dres, dx, dg, db, dxsum, rows, d, workspace,
                                  workspace_bytes, dxm, *drop);
}

extern "C" int db200_layernorm_divmax_bwd(db200_stream_t stream_, const void* dy, const void* x, const float* g,
                                          const float* mean, const float* rstd, const float* m, const void* dres,
                                          void* dx, void* dxm, float* dg, float* db, float* dxsum, int rows, int d,
                                          const db200_dropout* drop, void* workspace, int64_t workspace_bytes) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(m, DB200_E_INVALID, "layernorm_divmax_bwd: NULL m");
  if (!dropout_active(drop))
    return layernorm_bwd_impl<false, true>(stream, dy, x, g, mean, rstd, dres, dx, dg, db, dxsum, rows, d, workspace,
                                           workspace_bytes, nullptr, db200_dropout{}, m);
  DB200_REQUIRE(aligned16(dxm) && dxm, DB200_E_ALIGN, "layernorm_divmax_bwd: NULL or unaligned dxm");
  return layernorm_bwd_impl<true, true>(stream, dy, x, g, mean, rstd, dres, dx, dg, db, dxsum, rows, d, workspace,
                                        workspace_bytes, dxm, *drop, m);
}

extern "C" int db200_layernorm_bwd(db200_stream_t stream_, const void* dy, const void* x, const float* g,
                                   const float* mean, const float* rstd, const void* dres, void* dx, float* dg,
                                   float* db, int rows, int d, void* workspace, int64_t workspace_bytes) {
  return db200_layernorm_bwd_ex(stream_, dy, x, g, mean, rstd, dres, dx, dg, db, nullptr, rows, d, workspace,
                                workspace_bytes);
}

static int colsum_row_splits(int rows, int cols) {
  const int gx = (cols + 255) / 256;
  int gy = (sm_count() * 4 + gx - 1) / gx;
  if (gy > (rows + 7) / 8) gy = (rows + 7) / 8;
  return gy < 1 ? 1 : gy;
}

extern "C" int64_t db200_colsum_workspace_bytes(int rows, int cols) {
  return (int64_t)colsum_row_splits(rows, cols) * cols * (int64_t)sizeof(float);
}

extern "C" int db200_colsum_bf16(db200_stream_t stream_, const void* x, int64_t ld, int rows, int cols,
                                 float* out_accum, void* workspace, int64_t workspace_bytes) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(rows > 0 && cols > 0 && cols % 8 == 0 && ld % 8 == 0 && ld >= cols, DB200_E_INVALID,
                "colsum: need rows,cols > 0 and cols, ld multiples of 8 (got rows=%d cols=%d ld=%lld)", rows, cols,
                (long long)ld);
  DB200_REQUIRE(aligned16(x) && out_accum, DB200_E_ALIGN, "colsum: NULL or unaligned pointer");
  const int gx = (cols + 255) / 256;
  const int gy = colsum_row_splits(rows, cols);
  DB200_REQUIRE(workspace_ok(workspace, workspace_bytes, db200_colsum_workspace_bytes(rows, cols)), DB200_E_INVALID,
                "colsum: needs an aligned workspace of db200_colsum_workspace_bytes() bytes");
  float* ws = static_cast<float*>(workspace);
  colsum_kernel<<<dim3(gx, gy), 256, 0, stream>>>((const bf16*)x, ld, rows, cols, ws);
  const int rc = check_launch("colsum_kernel");
  if (rc != DB200_OK) return rc;
  return reduce_rows_add(stream, ws, gy, cols, out_accum);
}

extern "C" int db200_cast_f32_to_bf16(db200_stream_t stream_, const float* src, void* dst, size_t n) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (n == 0) return DB200_OK;
  DB200_REQUIRE(aligned16(src) && aligned16(dst) && src && dst, DB200_E_ALIGN, "cast: NULL or unaligned pointer");
  size_t blocks = (n / 8 + 255) / 256;
  if (blocks > sm_count() * 16) blocks = sm_count() * 16;
  if (blocks < 1) blocks = 1;
  cast_f32_bf16_kernel<<<(int)blocks, 256, 0, stream>>>(src, (bf16*)dst, n);
  return check_launch("cast_f32_bf16_kernel");
}
extern "C" int db200_cast_bf16_to_f32(db200_stream_t stream_, const void* src, float* dst, size_t n) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (n == 0) return DB200_OK;
  DB200_REQUIRE(aligned16(src) && aligned16(dst) && src && dst, DB200_E_ALIGN, "cast: NULL or unaligned pointer");
  size_t blocks = (n / 8 + 255) / 256;
  if (blocks > sm_count() * 16) blocks = sm_count() * 16;
  if (blocks < 1) blocks = 1;
  cast_bf16_f32_kernel<<<(int)blocks, 256, 0, stream>>>((const bf16*)src, dst, n);
  return check_launch("cast_bf16_f32_kernel");
}

// Segmented bf16 -> f32 gather: segment i copies len[i] elements from src + src_off[i] to dst + dst_off[i]
// (table = int64 triples {src_off, dst_off, len} in device memory).  One CTA per segment (grid-stride inside).
// Used by the optimiser-state-sharded (ZeRO-1) mode: after the all-gather of the bf16 parameters every rank rebuilds
// its compact fp32 copy of the vector parameters (LayerNorm gains / biases, all biases) in ONE launch.
__global__ void __launch_bounds__(256)
gather_cast_kernel(const bf16* __restrict__ src, float* __restrict__ dst, const long long* __restrict__ table) {
  const long long so = table[3 * blockIdx.x], d0 = table[3 * blockIdx.x + 1], n = table[3 * blockIdx.x + 2];
  for (long long i = threadIdx.x; i < n; i += 256) dst[d0 + i] = __bfloat162float(src[so + i]);
}

extern "C" int db200_gather_cast_bf16_f32(db200_stream_t stream_, const void* src, float* dst, const int64_t* table_dev,
                                          int n_segments) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (n_segments == 0) return DB200_OK;
  DB200_REQUIRE(src && dst && table_dev && n_segments > 0, DB200_E_INVALID, "gather_cast: bad arguments");
  gather_cast_kernel<<<n_segments, 256, 0, stream>>>((const bf16*)src, dst,
                                                      reinterpret_cast<const long long*>(table_dev));
  return check_launch("gather_cast_kernel");
}

extern "C" int db200_split_f32_to_bf16x2(db200_stream_t stream_, const float* src, void* hi, void* lo_or_null, size_t n) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (n == 0) return DB200_OK;
  DB200_REQUIRE(src && hi && aligned16(src) && aligned16(hi) && aligned16(lo_or_null), DB200_E_ALIGN,
                "split_f32: NULL or unaligned pointer");
  size_t blocks = (n / 8 + 255) / 256;
  if (blocks > sm_count() * 16) blocks = sm_count() * 16;
  if (blocks < 1) blocks = 1;
  split_f32_kernel<<<(int)blocks, 256, 0, stream>>>(src, (bf16*)hi, (bf16*)lo_or_null, n);
  return check_launch("split_f32_kernel");
}

extern "C" int64_t db200_ce_finish_workspace_bytes(int M) {
  return (int64_t)((M + CEF_ROWS - 1) / CEF_ROWS) * (int64_t)sizeof(float);
}

extern "C" int db200_ce_finish(db200_stream_t stream_, const float* part_max, const float* part_sum,
                               const float* label_logit, float* lse, float* loss_rows, float* loss_sum, int M,
                               int n_tiles, void* workspace, int64_t workspace_bytes) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(M > 0 && n_tiles > 0, DB200_E_INVALID, "ce_finish: M and n_tiles must be positive");
  DB200_REQUIRE(part_max && part_sum && label_logit && lse && loss_rows && loss_sum, DB200_E_INVALID,
                "ce_finish: NULL pointer");
  const int blocks = (M + CEF_ROWS - 1) / CEF_ROWS;
  DB200_REQUIRE(workspace_ok(workspace, workspace_bytes, db200_ce_finish_workspace_bytes(M)), DB200_E_INVALID,
                "ce_finish: needs an aligned workspace of db200_ce_finish_workspace_bytes() bytes");
  float* ws = static_cast<float*>(workspace);
  ce_finish_kernel<<<blocks, CEF_ROWS * CEF_GROUPS, 0, stream>>>(part_max, part_sum, label_logit, lse, loss_rows, ws, M,
                                                                 n_tiles);
  const int rc = check_launch("ce_finish_kernel");
  if (rc != DB200_OK) return rc;
  return reduce_rows_add(stream, ws, blocks, 1, loss_sum);
}

extern "C" int64_t db200_ce_finish_weighted_workspace_bytes(int M) {
  return (int64_t)((M + CEF_ROWS - 1) / CEF_ROWS) * 4 * (int64_t)sizeof(float);
}

extern "C" int db200_ce_finish_weighted(db200_stream_t stream_, const float* part_max, const float* part_sum,
                                        const float* label_logit, float* lse, float* loss_rows, float* sums, int M,
                                        int n_tiles, const db200_ce_weights* w, void* workspace,
                                        int64_t workspace_bytes) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(M > 0 && n_tiles > 0, DB200_E_INVALID, "ce_finish_weighted: M and n_tiles must be positive");
  DB200_REQUIRE(part_max && part_sum && label_logit && lse && loss_rows && sums, DB200_E_INVALID,
                "ce_finish_weighted: NULL pointer");
  const int rc0 = ce_weights_check(w, "ce_finish_weighted");
  if (rc0 != DB200_OK) return rc0;
  const int blocks = (M + CEF_ROWS - 1) / CEF_ROWS;
  DB200_REQUIRE(workspace_ok(workspace, workspace_bytes, db200_ce_finish_weighted_workspace_bytes(M)), DB200_E_INVALID,
                "ce_finish_weighted: needs an aligned workspace of db200_ce_finish_weighted_workspace_bytes() bytes");
  float* ws = static_cast<float*>(workspace);
  ce_finish_weighted_kernel<<<blocks, CEF_ROWS * CEF_GROUPS, 0, stream>>>(part_max, part_sum, label_logit, lse,
                                                                          loss_rows, ws, M, n_tiles, *w);
  const int rc = check_launch("ce_finish_weighted_kernel");
  if (rc != DB200_OK) return rc;
  return reduce_rows_add(stream, ws, blocks, 4, sums);
}
