// N4 — incremental (KV-cache) decoding kernels: the "is_incremental_inference" path the reference sketches in
// src/dalle_mtf/models.py:246-254, 281-285 (new k/v blended into the cached states at context.position - 1, the query of
// the current position attends to keys <= position) but never wires up (PREDICT raises NotImplementedError,
// src/model_fns.py:135-136).  All of it is HBM / latency bound work on B rows per step.
//
//   embed_fwd_at   x[b,:] = wte[ids[b],:] + wpe[pos,:]                     (models.py:186-219 at one position)
//   attn_decode    append this step's k,v to the cache at `pos`, then out[b,h,:] = softmax_{lo<=j<=pos}(scale q.k_j) v_j,
//                  lo = max(0, pos - radius + 1) (radius >= S: every key <= pos; a local layer, models.py:257-273: its window)
//                  fp32 scores / softmax, P rounded to bf16 for the PV product (same policy as attn.cu)
//                  AXIAL (row / column layers): over a key list, the text run [0, min(pos, TL - 1)] followed, for an
//                  image position (grid row r, column c), by row r's columns 0..c or column c's rows 0..r
//                  CONV (convolutional layers, kernel k): the text run followed by one run per row r' of the k x k
//                  window, max(0, r - k + 1) <= r' <= r, each over columns max(0, c - k + 1) .. c
//                  SPARSE (block-sparse layers): over the 16-key blocks listed for row block pos / 16, clipped at pos
//   sample_rows    idx = lo + argmax_{lo<=c<hi}(logits[c] * inv_temp + gumbel(u[c-lo]))   (first maximum; u NULL = greedy)
//   sample_rows_filtered   the same argmax restricted to the top-k / nucleus (top-p) set of logits * inv_temp
//   sample_rows_guided     either of the two over the classifier-free-guidance mix u + s (c - u) of a conditional
//                          and an unconditional row (the <true> instantiations); the draw goes to both rows' tokens
//   caption_next   after a draw into text column c: the prompt id below the row's prompt length, else the column's pad
//                  once column c - 1 or the draw is a padding token (caption completion)
//   onehot_rows    y[r, idx[r]-offset] = 1, 0 elsewhere (codebook lookup input for the VAE decoder, vae_tf/models.py:127)
#include "common.cuh"
#include "ptx.cuh"

namespace db200 {

// pos_dev != NULL: the position is read from device memory (CUDA-graph replay: one captured step serves every position)
// and the token of row b is ids[b * ld_ids + pos] (the [B][S] token matrix itself); else ids[b * ld_ids] at `pos`.
__global__ void embed_at_kernel(const int* __restrict__ ids, const bf16* __restrict__ wte, const bf16* __restrict__ wpe,
                                bf16* __restrict__ out, int d, int V, int pos, const int* __restrict__ pos_dev,
                                long long ld_ids) {
  const int b = blockIdx.x;
  if (pos_dev) pos = *pos_dev;
  int id = ids[b * ld_ids + (pos_dev ? pos : 0)];
  id = id < 0 ? 0 : (id >= V ? V - 1 : id);
  const bf16* w = wte + (long long)id * d;
  const bf16* p = wpe + (long long)pos * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x)
    out[(long long)b * d + i] = __float2bfloat16(__bfloat162float(w[i]) + __bfloat162float(p[i]));
}

// one CTA per (head, batch); 8 warps.  Keys are split over the warps in BOTH passes (scores, then P.V), a warp reads a
// whole cached row per instruction (dh * 2 contiguous bytes) and keeps four rows in flight: the per-thread serial walk
// over `pos` keys of the first version made generation latency-bound (~100 us per call at pos ~ 1000).
// Scores live in dynamic shared memory, indexed by j - lo (pos + 1 - lo floats, or min(S, radius) when the position is
// read on the device).
// AXIAL: scores are indexed by position in the key list: list entry j < n1 is key j (the text run), entry n1 + i is
// key ist + i * istr (the image run of the position's row or column); at most text_len + grid_w entries.
// CONV: the same text run; entry n1 + i is key ist + (i / m) grid_w + i % m (m window columns per row, ist the window's
// top-left key); at most text_len + min(k, grid_w)^2 entries.
// SPARSE: row g = pos / 16 of the block list (blocks + g * bpitch: a count, then ascending block indices <= g); entry
// j is key 16 bl[j / 16] + j % 16.  Only the last listed block can reach past pos, so the list holds 16 (count - 1) +
// min(16, pos - 16 last + 1) keys, at most pos + 1.
template <int DH, bool AXIAL = false, bool CONV = false, bool SPARSE = false>
__global__ void __launch_bounds__(256)
attn_decode_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ kc, bf16* __restrict__ vc, bf16* __restrict__ out,
                   int S, int H, int pos, float scale, const int* __restrict__ pos_dev, int radius, int text_len,
                   int grid_w, int axis, int kernel, const int* __restrict__ blocks, int bpitch) {
  static_assert(int(AXIAL) + int(CONV) + int(SPARSE) <= 1, "one key list");
  extern __shared__ float sc[];
  __shared__ float red[8];
  __shared__ float part[8][DH];
  if (pos_dev) pos = *pos_dev;
  constexpr int EPL = DH / 32;  // elements per lane (4 or 2): lane l owns [l * EPL, (l + 1) * EPL) of a row
  const int h = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bf16* q = qkv + ((long long)b * 3 + 0) * H * DH + (long long)h * DH;
  const bf16* k = qkv + ((long long)b * 3 + 1) * H * DH + (long long)h * DH;
  const bf16* v = qkv + ((long long)b * 3 + 2) * H * DH + (long long)h * DH;
  bf16* kcb = kc + ((long long)b * S * H + h) * DH;  // + j * H * DH
  bf16* vcb = vc + ((long long)b * S * H + h) * DH;
  const long long rs = (long long)H * DH;            // row stride of the caches
  for (int t = tid; t < DH; t += 256) {
    kcb[(long long)pos * rs + t] = k[t];
    vcb[(long long)pos * rs + t] = v[t];
  }
  float qr[EPL];
#pragma unroll
  for (int e = 0; e < EPL; ++e) qr[e] = __bfloat162float(q[lane * EPL + e]);
  __syncthreads();  // this block's own global writes are visible to it after the barrier
  const int lo = (AXIAL || CONV || SPARSE) ? 0 : max(0, pos - radius + 1);
  int n = pos + 1 - lo, n1 = 0, ist = 0, istr = 0, m = 1;
  if constexpr (AXIAL) {
    n1 = min(pos, text_len - 1) + 1;
    n = n1;
    if (pos >= text_len) {
      const int k = pos - text_len, r = k / grid_w, c = k % grid_w;
      ist = text_len + (axis ? c : r * grid_w);
      istr = axis ? grid_w : 1;
      n += (axis ? r : c) + 1;
    }
  }
  if constexpr (CONV) {
    n1 = min(pos, text_len - 1) + 1;
    n = n1;
    if (pos >= text_len) {
      const int k = pos - text_len, r = k / grid_w, c = k % grid_w;
      const int r0 = max(0, r - kernel + 1), c0 = max(0, c - kernel + 1);
      m = c - c0 + 1;
      ist = text_len + r0 * grid_w + c0;
      n += (r - r0 + 1) * m;
    }
  }
  const int* bl = nullptr;
  if constexpr (SPARSE) {
    const int* row = blocks + (long long)(pos >> 4) * bpitch;
    const int cnt = row[0];
    bl = row + 1;
    n = cnt > 0 ? 16 * (cnt - 1) + min(16, pos - 16 * bl[cnt - 1] + 1) : 0;
  }
  // key row of list entry j
  auto key = [&](int j) {
    if constexpr (SPARSE) return 16 * bl[j >> 4] + (j & 15);
    else if constexpr (CONV) return j < n1 ? j : ist + (j - n1) / m * grid_w + (j - n1) % m;
    else return AXIAL ? (j < n1 ? j : ist + (j - n1) * istr) : j;
  };
  const bf16* kw = kcb + (long long)lo * rs;         // key / value rows of the window: j - lo = 0 .. n - 1
  const bf16* vw = vcb + (long long)lo * rs;
  auto load_row = [&](const bf16* base, int j, float* o) {
    if (EPL == 4) {
      const uint2 u = *reinterpret_cast<const uint2*>(base + (long long)j * rs + lane * 4);
      const float2 a = unpack_bf16x2(u.x), c = unpack_bf16x2(u.y);
      o[0] = a.x; o[1] = a.y; o[2] = c.x; o[3] = c.y;
    } else {
      const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(base + (long long)j * rs + lane * 2));
      o[0] = a.x; o[1] = a.y;
    }
  };
  // ---- scores: warp w takes keys w, w + 8, ... four at a time
  float mx = -INFINITY;
  for (int j0 = warp; j0 < n; j0 += 32) {
    float kr[4][EPL], s[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (j0 + 8 * u < n) load_row(kw, key(j0 + 8 * u), kr[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      s[u] = 0.f;
      if (j0 + 8 * u < n) {
#pragma unroll
        for (int e = 0; e < EPL; ++e) s[u] += qr[e] * kr[u][e];
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float t = warp_sum(s[u]) * scale;
      if (j0 + 8 * u < n) {
        if (lane == 0) sc[j0 + 8 * u] = t;
        mx = fmaxf(mx, t);
      }
    }
  }
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int j = tid; j < n; j += 256) {
    const float p = __expf(sc[j] - mx);
    sum += p;
    sc[j] = __bfloat162float(__float2bfloat16(p));  // P goes through bf16 for the PV product, the sum does not
  }
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) sum += red[w];
  // ---- P.V: warp w accumulates its keys' contributions to all dh outputs, then the 8 partials are summed
  float acc[EPL];
#pragma unroll
  for (int e = 0; e < EPL; ++e) acc[e] = 0.f;
  for (int j0 = warp; j0 < n; j0 += 32) {
    float vr[4][EPL];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (j0 + 8 * u < n) load_row(vw, key(j0 + 8 * u), vr[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (j0 + 8 * u < n) {
        const float p = sc[j0 + 8 * u];
#pragma unroll
        for (int e = 0; e < EPL; ++e) acc[e] += p * vr[u][e];
      }
  }
#pragma unroll
  for (int e = 0; e < EPL; ++e) part[warp][lane * EPL + e] = acc[e];
  __syncthreads();
  const float inv = (SPARSE && sum == 0.f) ? 0.f : 1.f / sum;  // SPARSE: a row without keys gives 0
  for (int t = tid; t < DH; t += 256) {
    float o = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) o += part[w][t];
    out[((long long)b * H + h) * DH + t] = __float2bfloat16(o * inv);
  }
}

// The Gumbel-max perturbation x + g(u), g(u) = -log(-log u); the filtered sampler uses the same expression, so with its
// filter off it selects exactly what sample_rows_kernel selects.
__device__ __forceinline__ float gumbel_perturb(float x, float u) { return x + -logf(-logf(u)); }

// Classifier-free guidance: the combined logit u + s (c - u) of a conditional value c and an unconditional value u,
// rounded op by op (no FMA contraction), so a float32 host computation reproduces it bit for bit.
__device__ __forceinline__ float guided_logit(float c, float u, float s) {
  return __fadd_rn(u, __fmul_rn(s, __fsub_rn(c, u)));
}

// GUIDED: logits holds 2 * rows rows, the conditional ones first; row r's value of id c is guided_logit(row r,
// row rows + r, gscale), the noise has one row per pair, and the draw goes to column col of token rows r and rows + r.
// GUIDED = false is the plain sampler (rows and gscale unused).
template <bool GUIDED>
__global__ void __launch_bounds__(256)
sample_rows_kernel(const float* __restrict__ logits, const float* __restrict__ u, int* __restrict__ idx, long long ld,
                   int lo, int hi, float inv_temp, const int* __restrict__ pos_dev, long long ld_idx, int rows,
                   float gscale) {
  __shared__ float bv[8];
  __shared__ int bi[8];
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* row = logits + (long long)r * ld;
  const float* urow = GUIDED ? row + (long long)rows * ld : nullptr;
  const int n = hi - lo;
  float best = -INFINITY;
  int arg = 0x7fffffff;
  for (int c = tid; c < n; c += 256) {
    float x = (GUIDED ? guided_logit(row[lo + c], urow[lo + c], gscale) : row[lo + c]) * inv_temp;
    if (u) x = gumbel_perturb(x, u[(long long)r * n + c]);
    if (x > best || (x == best && c < arg)) { best = x; arg = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, arg, o);
    if (ov > best || (ov == best && oi < arg)) { best = ov; arg = oi; }
  }
  if (lane == 0) { bv[warp] = best; bi[warp] = arg; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < 8; ++w)
      if (bv[w] > best || (bv[w] == best && bi[w] < arg)) { best = bv[w]; arg = bi[w]; }
    const int id = lo + (arg == 0x7fffffff ? 0 : arg);  // all -inf / NaN row: first allowed id
    if (GUIDED) {
      const long long col = pos_dev ? *pos_dev + 1 : 0;
      idx[r * ld_idx + col] = id;
      idx[(rows + r) * ld_idx + col] = id;
    } else {
      // pos_dev != NULL (graph replay): the sample is the token of position *pos_dev + 1 of the [rows][ld_idx] matrix
      int* dst = pos_dev ? idx + r * ld_idx + (*pos_dev + 1) : idx + r;
      *dst = id;
    }
  }
}

// ---- top-k / nucleus (top-p) filtered sampling.  One CTA per row; the row's x = logits * inv_temp is staged in dynamic
// shared memory as order-preserving uint32 keys, so "x_a > x_b" is "key_a > key_b" and every kept set is an upper set
// of keys {key >= T}: the kernel finds T and then runs the Gumbel-max over the keys >= T.
//   top-k: T_k = the k-th largest key (ties at T_k all kept), by MSB-first radix select (8-bit digits, 4 passes of a
//          256-bin count histogram);
//   top-p: over the keys >= T_k, w = exp(x - max), Z = sum w; x is kept iff the mass strictly above it is < p * Z.
//          The same 4-pass descent over per-bin mass finds the smallest such key.  Masses are 64-bit fixed point
//          (2^-46 units) summed with integer atomics, so the kept set is the same on every run.
// NaN and -inf map to key 0 and are never kept; -0 is stored as +0 (the two compare equal, so must share a key);
// +inf entries, if any, are the only ones kept (the softmax mass is undefined there).
constexpr int SF_THREADS = 1024, SF_WARPS = SF_THREADS / 32;
constexpr int SF_SMEM_BYTES = 200 * 1024;                       // dynamic shared memory: one uint32 key per id
constexpr int SF_MAX_N = SF_SMEM_BYTES / 4;                      // 51 200 ids per row
constexpr uint32_t SF_KEY_PINF = 0xff800000u;                   // key of +inf
constexpr int SF_NONE = 256;                                    // histogram bin of ids a pass ignores

__device__ __forceinline__ uint32_t sf_key(float x) {
  if (!(x > -INFINITY)) return 0u;                              // NaN, -inf
  const uint32_t b = __float_as_uint(x == 0.f ? 0.f : x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ float sf_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Thread t < 256 passes v = the value of bin 255 - t and gets the total of the bins above that digit.  Called by every
// thread of the CTA (it synchronises); wtot holds 8 partials.
__device__ __forceinline__ unsigned long long sf_sum_above(unsigned long long v, unsigned long long* wtot) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  unsigned long long incl = 0;
  if (tid < 256) {
    incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) wtot[warp] = incl;
  }
  __syncthreads();
  if (tid < 256)
    for (int w = 0; w < warp; ++w) incl += wtot[w];
  return incl - v;
}

__device__ __forceinline__ uint32_t sf_block_sum(uint32_t v, uint32_t* red) {
  v = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t s = 0;
#pragma unroll 8
  for (int w = 0; w < SF_WARPS; ++w) s += red[w];
  __syncthreads();
  return s;
}

__device__ __forceinline__ uint32_t sf_block_max(uint32_t v, uint32_t* red) {
  v = __reduce_max_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t s = 0;
#pragma unroll 8
  for (int w = 0; w < SF_WARPS; ++w) s = max(s, red[w]);
  __syncthreads();
  return s;
}

__device__ __forceinline__ unsigned long long sf_mass(uint32_t k, float xmax) {
  return __float2ull_rn(expf(sf_value(k) - xmax) * 0x1p46f);  // w in (0, 1] -> [0, 2^46]
}

// GUIDED: the pair layout of sample_rows_kernel<true>; kept[r] counts the kept ids of pair r.
template <bool GUIDED>
__global__ void __launch_bounds__(SF_THREADS)
sample_rows_filtered_kernel(const float* __restrict__ logits, const float* __restrict__ u, int* __restrict__ idx,
                            int* __restrict__ kept, long long ld, int lo, int hi, float inv_temp, int top_k, float top_p,
                            const int* __restrict__ pos_dev, long long ld_idx, int rows, float gscale) {
  extern __shared__ uint32_t keys[];
  __shared__ uint32_t mlo[SF_NONE + 1], mhi[SF_NONE + 1];  // per-bin mass = mhi * 2^32 + mlo (no 64-bit smem atomics)
  __shared__ uint32_t cnt[SF_NONE + 1];
  __shared__ unsigned long long wtot[SF_WARPS];
  __shared__ uint32_t red[SF_WARPS];
  __shared__ int sel;
  __shared__ unsigned long long sel_above;
  __shared__ float bv[SF_WARPS];
  __shared__ int bi[SF_WARPS];
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* row = logits + (long long)r * ld;
  const float* urow = GUIDED ? row + (long long)rows * ld : nullptr;
  const int n = hi - lo;

  uint32_t nv = 0, ninf = 0, kmax = 0;
  for (int c = tid; c < n; c += SF_THREADS) {
    const uint32_t k = sf_key((GUIDED ? guided_logit(row[lo + c], urow[lo + c], gscale) : row[lo + c]) * inv_temp);
    keys[c] = k;
    nv += k != 0;
    ninf += k == SF_KEY_PINF;
    kmax = max(kmax, k);
  }
  nv = sf_block_sum(nv, red);      // (the barriers inside also publish keys[])
  ninf = sf_block_sum(ninf, red);
  kmax = sf_block_max(kmax, red);

  uint32_t T = 1;                  // smallest kept key; 0 (NaN, -inf) is never kept
  if (nv == 0) {
    T = 0xffffffffu;               // nothing is kept: the largest key in use is SF_KEY_PINF
  } else if (ninf > 0) {
    T = SF_KEY_PINF;
  } else {
    if (top_k > 0 && (uint32_t)top_k < nv) {
      // radix select of the k-th largest key: `rem` ids are still to be counted from the top inside `prefix`
      uint32_t prefix = 0, rem = (uint32_t)top_k;
      for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        const uint32_t himask = pass == 0 ? 0u : ~0u << (shift + 8);
        for (int b = tid; b <= SF_NONE; b += SF_THREADS) cnt[b] = 0;
        __syncthreads();
        for (int c0 = 0; c0 < n; c0 += SF_THREADS) {   // uniform trip count: whole warps take part in the match
          const int c = c0 + tid;
          const uint32_t k = c < n ? keys[c] : 0u;
          const int d = (k != 0 && (k & himask) == prefix) ? (int)((k >> shift) & 255u) : SF_NONE;
          if (!__any_sync(0xffffffffu, d != SF_NONE)) continue;
          const unsigned peers = __match_any_sync(0xffffffffu, d);
          if (d != SF_NONE && lane == __ffs(peers) - 1) atomicAdd(&cnt[d], (uint32_t)__popc(peers));
        }
        __syncthreads();
        const unsigned long long above = sf_sum_above(tid < 256 ? cnt[255 - tid] : 0u, wtot);
        if (tid < 256 && above < rem && above + cnt[255 - tid] >= rem) {
          sel = 255 - tid;
          sel_above = above;
        }
        __syncthreads();
        prefix |= (uint32_t)sel << shift;
        rem -= (uint32_t)sel_above;
        __syncthreads();
      }
      T = prefix;
    }
    if (top_p < 1.f) {
      const float xmax = sf_value(kmax);
      unsigned long long z = 0;
      for (int c = tid; c < n; c += SF_THREADS) {
        const uint32_t k = keys[c];
        if (k >= T) z += sf_mass(k, xmax);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
      if (lane == 0) wtot[warp] = z;
      __syncthreads();
      z = 0;
      for (int w = 0; w < SF_WARPS; ++w) z += wtot[w];
      __syncthreads();
      const double pz = (double)top_p * (double)z;
      // descent: `above` = mass of the kept-candidate ids (keys >= T) whose key lies above `prefix`
      uint32_t prefix = 0;
      unsigned long long above = 0;
      for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        const uint32_t himask = pass == 0 ? 0u : ~0u << (shift + 8);
        for (int b = tid; b <= SF_NONE; b += SF_THREADS) { cnt[b] = 0; mlo[b] = 0; mhi[b] = 0; }
        if (tid == 0) sel = -1;
        __syncthreads();
        for (int c0 = 0; c0 < n; c0 += SF_THREADS) {
          const int c = c0 + tid;
          const uint32_t k = c < n ? keys[c] : 0u;
          const int d = (k >= T && (k & himask) == prefix) ? (int)((k >> shift) & 255u) : SF_NONE;
          if (!__any_sync(0xffffffffu, d != SF_NONE)) continue;
          const unsigned long long w = d != SF_NONE ? sf_mass(k, xmax) : 0ull;
          const unsigned peers = __match_any_sync(0xffffffffu, d);
          // per-digit warp sums of the two 23-bit halves of w (at most 32 * 2^23 each: no overflow in 32 bits)
          const uint32_t wlo = __reduce_add_sync(peers, (uint32_t)(w & 0x7fffffu));
          const uint32_t whi = __reduce_add_sync(peers, (uint32_t)(w >> 23));
          if (d != SF_NONE && lane == __ffs(peers) - 1) {
            const unsigned long long add = ((unsigned long long)whi << 23) + wlo;
            const uint32_t alo = (uint32_t)add, old = atomicAdd(&mlo[d], alo);
            atomicAdd(&mhi[d], (uint32_t)(add >> 32) + (old + alo < old ? 1u : 0u));   // carry out of the low word
            atomicAdd(&cnt[d], (uint32_t)__popc(peers));
          }
        }
        __syncthreads();
        // the largest key of bin 255 - tid has mass above + (bins above it) strictly above it: the lowest non-empty
        // bin where that is < p * Z holds T_p
        const unsigned long long in =
            sf_sum_above(tid < 256 ? ((unsigned long long)mhi[255 - tid] << 32) + mlo[255 - tid] : 0ull, wtot);
        if (tid < 256 && cnt[255 - tid] > 0 && (double)(above + in) < pz) atomicMax(&sel, tid);
        __syncthreads();
        if (tid == sel) sel_above = in;
        __syncthreads();
        prefix |= (uint32_t)(255 - sel) << shift;
        above += sel_above;
        __syncthreads();
      }
      T = prefix;
    }
  }

  // Gumbel-max over the kept ids; first index on ties
  float best = -INFINITY;
  int arg = 0x7fffffff;
  uint32_t nk = 0;
  for (int c = tid; c < n; c += SF_THREADS) {
    const uint32_t k = keys[c];
    if (k < T) continue;
    ++nk;
    float x = sf_value(k);
    if (u) x = gumbel_perturb(x, u[(long long)r * n + c]);
    if (x > best || (x == best && c < arg)) { best = x; arg = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, arg, o);
    if (ov > best || (ov == best && oi < arg)) { best = ov; arg = oi; }
  }
  if (lane == 0) { bv[warp] = best; bi[warp] = arg; }
  nk = sf_block_sum(nk, red);
  if (tid == 0) {
    for (int w = 1; w < SF_WARPS; ++w)
      if (bv[w] > best || (bv[w] == best && bi[w] < arg)) { best = bv[w]; arg = bi[w]; }
    const int id = lo + (arg == 0x7fffffff ? 0 : arg);  // no finite id: first allowed id
    if (GUIDED) {
      const long long col = pos_dev ? *pos_dev + 1 : 0;
      idx[r * ld_idx + col] = id;
      idx[(rows + r) * ld_idx + col] = id;
    } else {
      int* dst = pos_dev ? idx + r * ld_idx + (*pos_dev + 1) : idx + r;
      *dst = id;
    }
    if (kept) kept[r] = (int)nk;
  }
}

__global__ void incr_i32_kernel(int* p, int delta) { *p += delta; }

// ---- caption completion: finishes column c = pos + 1 of every row of the [rows][ld] token matrix after a draw has
// been written there.  Row b keeps its prompt below lens[b]; past it a padding token in column c - 1 or drawn in column
// c ends the caption: column c becomes c's pad (pad_base + c with per-position padding, else padding_id).  Integer
// arithmetic only, one thread per row.
__global__ void __launch_bounds__(128)
caption_next_kernel(int* __restrict__ tokens, long long ld, const int* __restrict__ prefix, long long ld_prefix,
                    const int* __restrict__ lens, int rows, int text_len, int text_vocab, int padding_id, int pad_base,
                    int pos, const int* __restrict__ pos_dev) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= rows) return;
  const int c = (pos_dev ? *pos_dev : pos) + 1;
  if (c < 1 || c >= text_len) return;
  int* row = tokens + b * ld;
  if (c < lens[b]) {
    row[c] = prefix[b * ld_prefix + c];
    return;
  }
  auto is_pad = [&](int id) { return id == padding_id || (pad_base >= 0 && id >= text_vocab); };
  if (is_pad(row[c - 1]) || is_pad(row[c])) row[c] = pad_base >= 0 ? pad_base + c : padding_id;
}

__global__ void onehot_rows_kernel(const int* __restrict__ idx, float* __restrict__ y, int K, int offset) {
  const int r = blockIdx.x;
  const int hot = idx[r] - offset;
  for (int c = threadIdx.x; c < K; c += blockDim.x) y[(long long)r * K + c] = (c == hot) ? 1.f : 0.f;
}

// ---- prompt prefill hand-off.  Pure copies in 16-byte vectors (8 bf16): one source vector is read once and stored
// into every replica, so the source traffic does not grow with `rep`.
// kv_cache_fill: vector c of (b, p, k|v) of qkv [B][P][3][H*dh/8] -> caches [B*rep][S_cache][H*dh/8] at position p.
__global__ void __launch_bounds__(256)
kv_cache_fill_kernel(const uint4* __restrict__ qkv, uint4* __restrict__ kc, uint4* __restrict__ vc, int P, int S_cache,
                     int rep, int n16, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % n16);
    long long t = i / n16;
    const int kv = (int)(t & 1);
    t >>= 1;
    const int p = (int)(t % P);
    const long long b = t / P;
    const uint4 v = qkv[((b * P + p) * 3 + 1 + kv) * n16 + c];
    uint4* dst = kv ? vc : kc;
    for (int r = 0; r < rep; ++r) dst[((b * rep + r) * S_cache + p) * n16 + c] = v;
  }
}

// rows_repeat: dst row b * rep + r = src row b (row stride ld16 vectors), d16 vectors per row.
__global__ void __launch_bounds__(256)
rows_repeat_kernel(const uint4* __restrict__ src, long long ld16, uint4* __restrict__ dst, int d16, int rep,
                   long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % d16);
    const long long b = i / d16;
    const uint4 v = src[b * ld16 + c];
    for (int r = 0; r < rep; ++r) dst[(b * rep + r) * d16 + c] = v;
  }
}

}  // namespace db200

using namespace db200;

extern "C" int db200_embed_fwd_at(db200_stream_t stream_, const int32_t* ids, const void* wte, const void* wpe,
                                  void* out, int B, int d, int V, int n_pos, int pos) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(ids && wte && wpe && out, DB200_E_INVALID, "embed_fwd_at: null pointer");
  DB200_REQUIRE(B > 0 && d > 0 && V > 0 && pos >= 0 && pos < n_pos, DB200_E_INVALID,
                "embed_fwd_at: B %d d %d V %d pos %d of %d", B, d, V, pos, n_pos);
  embed_at_kernel<<<B, 256, 0, stream>>>(ids, static_cast<const bf16*>(wte), static_cast<const bf16*>(wpe),
                                         static_cast<bf16*>(out), d, V, pos, nullptr, 1);
  return check_launch("embed_at_kernel");
}

// ---- device-side position variants (CUDA-graph replay of the per-position step): `pos_dev` points at one int32 in
// device memory that the caller advances with db200_incr_i32 between replays; `tokens` is the [B][ld] token matrix.
extern "C" int db200_embed_fwd_at_dev(db200_stream_t stream_, const int32_t* tokens, long long ld, const void* wte,
                                      const void* wpe, void* out, int B, int d, int V, const int32_t* pos_dev) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(tokens && wte && wpe && out && pos_dev && B > 0 && d > 0 && V > 0 && ld > 0, DB200_E_INVALID,
                "embed_fwd_at_dev: bad argument");
  embed_at_kernel<<<B, 256, 0, stream>>>(tokens, static_cast<const bf16*>(wte), static_cast<const bf16*>(wpe),
                                         static_cast<bf16*>(out), d, V, 0, pos_dev, ld);
  return check_launch("embed_at_kernel");
}

extern "C" int db200_incr_i32(db200_stream_t stream_, int32_t* p, int delta) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(p, DB200_E_INVALID, "incr_i32: null pointer");
  incr_i32_kernel<<<1, 1, 0, stream>>>(p, delta);
  return check_launch("incr_i32_kernel");
}

// pos_dev == NULL: position `pos` (scores need min(pos + 1, radius) floats of shared memory); else the position is read
// on the device and shared memory is sized for min(S, radius) keys.  radius >= S: every key <= pos.
// axis >= 0: an axial layer (attn_decode_kernel<DH, true>, radius unused): the key list of `pos` (text_len + grid_w
// floats when the position is read on the device).
// kernel >= 1: a convolutional layer (attn_decode_kernel<DH, false, true>, radius and axis unused): the key list of
// `pos` (text_len + kernel min(kernel, grid_w) floats when the position is read on the device).
// blocks != NULL: a block-sparse layer (attn_decode_kernel<DH, false, false, true>, radius S): the keys of the blocks
// listed for pos / 16, at most as many as a global layer's.
static int attn_decode_launch(cudaStream_t stream, const void* qkv_step, void* k_cache, void* v_cache, void* out, int B,
                              int S, int H, int dh, int pos, float scale, const int32_t* pos_dev, int radius,
                              int text_len = 0, int grid_w = 1, int axis = -1, int kernel = 0,
                              const int32_t* blocks = nullptr, int bpitch = 0) {
  DB200_REQUIRE(qkv_step && k_cache && v_cache && out, DB200_E_INVALID, "attn_decode: null pointer");
  DB200_REQUIRE(B > 0 && H > 0 && S > 0 && pos >= 0 && pos < S, DB200_E_INVALID, "attn_decode: B %d H %d pos %d of %d",
                B, H, pos, S);
  DB200_REQUIRE(radius >= 1, DB200_E_INVALID, "attn_decode: radius %d < 1", radius);
  DB200_REQUIRE(dh == 64 || dh == 128, DB200_E_UNSUPPORTED, "attn_decode: head_dim %d not in {64,128}", dh);
  const bool axial = axis >= 0, conv = kernel >= 1;
  size_t keys = (size_t)min(pos_dev ? S : pos + 1, radius);
  if (conv) {
    if (pos_dev) {
      keys = (size_t)min((long long)S, (long long)text_len + (long long)kernel * min(kernel, grid_w));
    } else {
      const int k = pos - text_len, r = k / grid_w, c = k % grid_w;
      keys = (size_t)(min(pos, text_len - 1) + 1) +
             (k >= 0 ? (size_t)(r - max(0, r - kernel + 1) + 1) * (size_t)(c - max(0, c - kernel + 1) + 1) : 0);
    }
  }
  if (axial) {
    if (pos_dev) {
      keys = (size_t)min((long long)S, (long long)text_len + grid_w);
    } else {
      const int k = pos - text_len;
      keys = (size_t)(min(pos, text_len - 1) + 1) + (k >= 0 ? (size_t)((axis ? k / grid_w : k % grid_w) + 1) : 0);
    }
  }
  DB200_REQUIRE(keys * 4 <= 200 * 1024, DB200_E_UNSUPPORTED, "attn_decode: %zu keys exceed shared memory", keys);
  const size_t smem = keys * sizeof(float);
  dim3 grid(H, B);
  static const cudaError_t a128 = cudaFuncSetAttribute(attn_decode_kernel<128>,
                                                       cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  static const cudaError_t a64 = cudaFuncSetAttribute(attn_decode_kernel<64>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  static const cudaError_t x128 = cudaFuncSetAttribute(attn_decode_kernel<128, true>,
                                                       cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  static const cudaError_t x64 = cudaFuncSetAttribute(attn_decode_kernel<64, true>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  DB200_CUDA(a128);
  DB200_CUDA(a64);
  static const cudaError_t c128 = cudaFuncSetAttribute(attn_decode_kernel<128, false, true>,
                                                       cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  static const cudaError_t c64 = cudaFuncSetAttribute(attn_decode_kernel<64, false, true>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  DB200_CUDA(x128);
  DB200_CUDA(x64);
  DB200_CUDA(c128);
  DB200_CUDA(c64);
  static const cudaError_t s128 = cudaFuncSetAttribute(attn_decode_kernel<128, false, false, true>,
                                                       cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  static const cudaError_t s64 = cudaFuncSetAttribute(attn_decode_kernel<64, false, false, true>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  DB200_CUDA(s128);
  DB200_CUDA(s64);
  const bool sparse = blocks != nullptr;
  auto fn = dh == 128 ? (sparse ? attn_decode_kernel<128, false, false, true>
                         : conv ? attn_decode_kernel<128, false, true>
                                : axial ? attn_decode_kernel<128, true> : attn_decode_kernel<128>)
                      : (sparse ? attn_decode_kernel<64, false, false, true>
                         : conv ? attn_decode_kernel<64, false, true>
                                : axial ? attn_decode_kernel<64, true> : attn_decode_kernel<64>);
  fn<<<grid, 256, smem, stream>>>(static_cast<const bf16*>(qkv_step), static_cast<bf16*>(k_cache),
                                  static_cast<bf16*>(v_cache), static_cast<bf16*>(out), S, H, pos, scale, pos_dev,
                                  radius, text_len, grid_w, axis, kernel, blocks, bpitch);
  return check_launch("attn_decode_kernel");
}

extern "C" int db200_attn_decode(db200_stream_t stream_, const void* qkv_step, void* k_cache, void* v_cache, void* out,
                                 int B, int S, int H, int dh, int pos, float scale) {
  return attn_decode_launch(static_cast<cudaStream_t>(stream_), qkv_step, k_cache, v_cache, out, B, S, H, dh, pos, scale,
                            nullptr, S);
}

extern "C" int db200_attn_decode_dev(db200_stream_t stream_, const void* qkv_step, void* k_cache, void* v_cache,
                                     void* out, int B, int S, int H, int dh, const int32_t* pos_dev, float scale) {
  DB200_REQUIRE(pos_dev, DB200_E_INVALID, "attn_decode_dev: null position pointer");
  return attn_decode_launch(static_cast<cudaStream_t>(stream_), qkv_step, k_cache, v_cache, out, B, S, H, dh, 0, scale,
                            pos_dev, S);
}

// local layers (src/dalle_mtf/models.py:257-273): the query of `pos` attends to keys [max(0, pos - radius + 1), pos]
extern "C" int db200_attn_decode_local(db200_stream_t stream_, const void* qkv_step, void* k_cache, void* v_cache,
                                       void* out, int B, int S, int H, int dh, int pos, int radius, float scale) {
  return attn_decode_launch(static_cast<cudaStream_t>(stream_), qkv_step, k_cache, v_cache, out, B, S, H, dh, pos, scale,
                            nullptr, radius);
}

extern "C" int db200_attn_decode_local_dev(db200_stream_t stream_, const void* qkv_step, void* k_cache, void* v_cache,
                                           void* out, int B, int S, int H, int dh, const int32_t* pos_dev, int radius,
                                           float scale) {
  DB200_REQUIRE(pos_dev, DB200_E_INVALID, "attn_decode_local_dev: null position pointer");
  return attn_decode_launch(static_cast<cudaStream_t>(stream_), qkv_step, k_cache, v_cache, out, B, S, H, dh, 0, scale,
                            pos_dev, radius);
}

// axial layers (row: axis 0, column: axis 1): the query of `pos` attends to the text keys [0, min(pos, text_len - 1)]
// and, at an image position (grid row r, column c), to row r's columns 0..c or column c's rows 0..r
static int axial_decode_args_ok(const char* fn, int S, int text_len, int grid_w, int axis) {
  DB200_REQUIRE(axis == 0 || axis == 1, DB200_E_INVALID, "%s: axis %d not 0 (row) or 1 (column)", fn, axis);
  DB200_REQUIRE(grid_w >= 1 && text_len >= 0, DB200_E_INVALID, "%s: grid_w %d < 1 or text_len %d < 0", fn, grid_w,
                text_len);
  DB200_REQUIRE((long long)S <= (long long)text_len + (long long)grid_w * grid_w, DB200_E_INVALID,
                "%s: S %d exceeds text_len %d + grid_w^2 (%d^2)", fn, S, text_len, grid_w);
  return DB200_OK;
}

extern "C" int db200_attn_decode_axial(db200_stream_t stream_, const void* qkv_step, void* k_cache, void* v_cache,
                                       void* out, int B, int S, int H, int dh, int pos, int text_len, int grid_w,
                                       int axis, float scale) {
  const int rc = axial_decode_args_ok("attn_decode_axial", S, text_len, grid_w, axis);
  if (rc != DB200_OK) return rc;
  return attn_decode_launch(static_cast<cudaStream_t>(stream_), qkv_step, k_cache, v_cache, out, B, S, H, dh, pos, scale,
                            nullptr, S, text_len, grid_w, axis);
}

extern "C" int db200_attn_decode_axial_dev(db200_stream_t stream_, const void* qkv_step, void* k_cache, void* v_cache,
                                           void* out, int B, int S, int H, int dh, const int32_t* pos_dev,
                                           int text_len, int grid_w, int axis, float scale) {
  DB200_REQUIRE(pos_dev, DB200_E_INVALID, "attn_decode_axial_dev: null position pointer");
  const int rc = axial_decode_args_ok("attn_decode_axial_dev", S, text_len, grid_w, axis);
  if (rc != DB200_OK) return rc;
  return attn_decode_launch(static_cast<cudaStream_t>(stream_), qkv_step, k_cache, v_cache, out, B, S, H, dh, 0, scale,
                            pos_dev, S, text_len, grid_w, axis);
}

// convolutional layers: the query of `pos` attends to the text keys [0, min(pos, text_len - 1)] and, at an image
// position (grid row r, column c), to the k x k window of keys at rows (r - kernel, r] and columns (c - kernel, c]
static int conv_decode_args_ok(const char* fn, int S, int text_len, int grid_w, int kernel) {
  DB200_REQUIRE(kernel >= 1, DB200_E_INVALID, "%s: kernel %d < 1", fn, kernel);
  DB200_REQUIRE(grid_w >= 1 && text_len >= 0, DB200_E_INVALID, "%s: grid_w %d < 1 or text_len %d < 0", fn, grid_w,
                text_len);
  DB200_REQUIRE((long long)S <= (long long)text_len + (long long)grid_w * grid_w, DB200_E_INVALID,
                "%s: S %d exceeds text_len %d + grid_w^2 (%d^2)", fn, S, text_len, grid_w);
  return DB200_OK;
}

extern "C" int db200_attn_decode_conv(db200_stream_t stream_, const void* qkv_step, void* k_cache, void* v_cache,
                                      void* out, int B, int S, int H, int dh, int pos, int text_len, int grid_w,
                                      int kernel, float scale) {
  const int rc = conv_decode_args_ok("attn_decode_conv", S, text_len, grid_w, kernel);
  if (rc != DB200_OK) return rc;
  return attn_decode_launch(static_cast<cudaStream_t>(stream_), qkv_step, k_cache, v_cache, out, B, S, H, dh, pos, scale,
                            nullptr, S, text_len, grid_w, -1, kernel);
}

extern "C" int db200_attn_decode_conv_dev(db200_stream_t stream_, const void* qkv_step, void* k_cache, void* v_cache,
                                          void* out, int B, int S, int H, int dh, const int32_t* pos_dev, int text_len,
                                          int grid_w, int kernel, float scale) {
  DB200_REQUIRE(pos_dev, DB200_E_INVALID, "attn_decode_conv_dev: null position pointer");
  const int rc = conv_decode_args_ok("attn_decode_conv_dev", S, text_len, grid_w, kernel);
  if (rc != DB200_OK) return rc;
  return attn_decode_launch(static_cast<cudaStream_t>(stream_), qkv_step, k_cache, v_cache, out, B, S, H, dh, 0, scale,
                            pos_dev, S, text_len, grid_w, -1, kernel);
}

// block-sparse layers: the query of `pos` attends to the keys of the 16-key blocks listed in row pos / 16 of `blocks`
extern "C" int db200_attn_decode_block_sparse(db200_stream_t stream_, const void* qkv_step, void* k_cache,
                                              void* v_cache, void* out, int B, int S, int H, int dh, int pos,
                                              const int32_t* blocks, int blocks_pitch, float scale) {
  DB200_REQUIRE(blocks && blocks_pitch >= (S + 15) / 16 + 1, DB200_E_INVALID,
                "attn_decode_block_sparse: NULL block table or pitch %d < ceil(S / 16) + 1 for S %d", blocks_pitch, S);
  return attn_decode_launch(static_cast<cudaStream_t>(stream_), qkv_step, k_cache, v_cache, out, B, S, H, dh, pos, scale,
                            nullptr, S, 0, 1, -1, 0, blocks, blocks_pitch);
}

extern "C" int db200_attn_decode_block_sparse_dev(db200_stream_t stream_, const void* qkv_step, void* k_cache,
                                                  void* v_cache, void* out, int B, int S, int H, int dh,
                                                  const int32_t* pos_dev, const int32_t* blocks, int blocks_pitch,
                                                  float scale) {
  DB200_REQUIRE(pos_dev, DB200_E_INVALID, "attn_decode_block_sparse_dev: null position pointer");
  DB200_REQUIRE(blocks && blocks_pitch >= (S + 15) / 16 + 1, DB200_E_INVALID,
                "attn_decode_block_sparse_dev: NULL block table or pitch %d < ceil(S / 16) + 1 for S %d", blocks_pitch,
                S);
  return attn_decode_launch(static_cast<cudaStream_t>(stream_), qkv_step, k_cache, v_cache, out, B, S, H, dh, 0, scale,
                            pos_dev, S, 0, 1, -1, 0, blocks, blocks_pitch);
}

extern "C" int db200_sample_rows(db200_stream_t stream_, const float* logits, const float* u_or_null, int32_t* idx,
                                 int rows, long long ld, int lo, int hi, float inv_temp) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(logits && idx, DB200_E_INVALID, "sample_rows: null pointer");
  DB200_REQUIRE(rows > 0 && lo >= 0 && hi > lo && hi <= ld, DB200_E_INVALID, "sample_rows: rows %d range [%d,%d) ld %lld",
                rows, lo, hi, ld);
  DB200_REQUIRE(inv_temp > 0.f, DB200_E_INVALID, "sample_rows: inv_temp must be positive");
  sample_rows_kernel<false><<<rows, 256, 0, stream>>>(logits, u_or_null, idx, ld, lo, hi, inv_temp, nullptr, 1, 0, 0.f);
  return check_launch("sample_rows_kernel");
}

// graph-replay variant: the sample of row r becomes tokens[r * ld_tokens + *pos_dev + 1]
extern "C" int db200_sample_rows_at(db200_stream_t stream_, const float* logits, const float* u_or_null,
                                    int32_t* tokens, long long ld_tokens, int rows, long long ld, int lo, int hi,
                                    float inv_temp, const int32_t* pos_dev) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(logits && tokens && pos_dev, DB200_E_INVALID, "sample_rows_at: null pointer");
  DB200_REQUIRE(rows > 0 && lo >= 0 && hi > lo && hi <= ld && inv_temp > 0.f, DB200_E_INVALID,
                "sample_rows_at: rows %d range [%d,%d) ld %lld", rows, lo, hi, ld);
  sample_rows_kernel<false><<<rows, 256, 0, stream>>>(logits, u_or_null, tokens, ld, lo, hi, inv_temp, pos_dev,
                                                      ld_tokens, 0, 0.f);
  return check_launch("sample_rows_kernel");
}

// guided: rows pairs, logits [2 * rows][ld] (sample_rows_kernel<true>)
static int sample_rows_filtered_launch(cudaStream_t stream, const float* logits, const float* u, int32_t* idx,
                                       int32_t* kept, int rows, long long ld, int lo, int hi, float inv_temp, int top_k,
                                       float top_p, const int32_t* pos_dev, long long ld_idx, bool guided = false,
                                       float gscale = 0.f) {
  DB200_REQUIRE(rows > 0 && lo >= 0 && hi > lo && hi <= ld, DB200_E_INVALID,
                "sample_rows_filtered: rows %d range [%d,%d) ld %lld", rows, lo, hi, ld);
  DB200_REQUIRE(inv_temp > 0.f, DB200_E_INVALID, "sample_rows_filtered: inv_temp must be positive");
  DB200_REQUIRE(top_k >= 0, DB200_E_INVALID, "sample_rows_filtered: top_k %d < 0", top_k);
  DB200_REQUIRE(top_p > 0.f && top_p <= 1.f, DB200_E_INVALID, "sample_rows_filtered: top_p %g outside (0, 1]",
                (double)top_p);
  DB200_REQUIRE(hi - lo <= SF_MAX_N, DB200_E_UNSUPPORTED, "sample_rows_filtered: %d ids exceed the %d one CTA holds",
                hi - lo, SF_MAX_N);
  static const cudaError_t attr = cudaFuncSetAttribute(sample_rows_filtered_kernel<false>,
                                                       cudaFuncAttributeMaxDynamicSharedMemorySize, SF_SMEM_BYTES);
  static const cudaError_t attr_g = cudaFuncSetAttribute(sample_rows_filtered_kernel<true>,
                                                         cudaFuncAttributeMaxDynamicSharedMemorySize, SF_SMEM_BYTES);
  DB200_CUDA(attr);
  DB200_CUDA(attr_g);
  const size_t smem = (size_t)(hi - lo) * sizeof(uint32_t);
  if (guided)
    sample_rows_filtered_kernel<true><<<rows, SF_THREADS, smem, stream>>>(logits, u, idx, kept, ld, lo, hi, inv_temp,
                                                                          top_k, top_p, pos_dev, ld_idx, rows, gscale);
  else
    sample_rows_filtered_kernel<false><<<rows, SF_THREADS, smem, stream>>>(logits, u, idx, kept, ld, lo, hi, inv_temp,
                                                                           top_k, top_p, pos_dev, ld_idx, 0, 0.f);
  return check_launch("sample_rows_filtered_kernel");
}

extern "C" int db200_sample_rows_filtered(db200_stream_t stream_, const float* logits, const float* u_or_null,
                                          int32_t* idx, int32_t* kept_or_null, int rows, long long ld, int lo, int hi,
                                          float inv_temp, int top_k, float top_p) {
  DB200_REQUIRE(logits && idx, DB200_E_INVALID, "sample_rows_filtered: null pointer");
  return sample_rows_filtered_launch(static_cast<cudaStream_t>(stream_), logits, u_or_null, idx, kept_or_null, rows, ld,
                                     lo, hi, inv_temp, top_k, top_p, nullptr, 1);
}

// graph-replay variant: the sample of row r becomes tokens[r * ld_tokens + *pos_dev + 1]
extern "C" int db200_sample_rows_filtered_at(db200_stream_t stream_, const float* logits, const float* u_or_null,
                                             int32_t* tokens, long long ld_tokens, int32_t* kept_or_null, int rows,
                                             long long ld, int lo, int hi, float inv_temp, int top_k, float top_p,
                                             const int32_t* pos_dev) {
  DB200_REQUIRE(logits && tokens && pos_dev, DB200_E_INVALID, "sample_rows_filtered_at: null pointer");
  return sample_rows_filtered_launch(static_cast<cudaStream_t>(stream_), logits, u_or_null, tokens, kept_or_null, rows,
                                     ld, lo, hi, inv_temp, top_k, top_p, pos_dev, ld_tokens);
}

// classifier-free guidance over `rows` (conditional, unconditional) pairs; the unfiltered kernel when no filter applies
extern "C" int db200_sample_rows_guided(db200_stream_t stream_, const float* logits, long long ld,
                                        const float* u_or_null, int32_t* tokens, long long ld_tokens,
                                        int32_t* kept_or_null, int rows, int lo, int hi, float inv_temp,
                                        float guidance_scale, int top_k, float top_p, const int32_t* pos_dev_or_null) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(logits && tokens, DB200_E_INVALID, "sample_rows_guided: null pointer");
  DB200_REQUIRE(ld_tokens > 0, DB200_E_INVALID, "sample_rows_guided: ld_tokens %lld", ld_tokens);
  DB200_REQUIRE(isfinite(guidance_scale) && guidance_scale >= 0.f, DB200_E_INVALID,
                "sample_rows_guided: guidance_scale %g must be finite and >= 0", (double)guidance_scale);
  if (top_k != 0 || top_p != 1.f)
    return sample_rows_filtered_launch(stream, logits, u_or_null, tokens, kept_or_null, rows, ld, lo, hi, inv_temp,
                                       top_k, top_p, pos_dev_or_null, ld_tokens, true, guidance_scale);
  DB200_REQUIRE(rows > 0 && lo >= 0 && hi > lo && hi <= ld, DB200_E_INVALID,
                "sample_rows_guided: rows %d range [%d,%d) ld %lld", rows, lo, hi, ld);
  DB200_REQUIRE(inv_temp > 0.f, DB200_E_INVALID, "sample_rows_guided: inv_temp must be positive");
  DB200_REQUIRE(!kept_or_null, DB200_E_INVALID, "sample_rows_guided: kept counts need an active top_k / top_p filter");
  sample_rows_kernel<true><<<rows, 256, 0, stream>>>(logits, u_or_null, tokens, ld, lo, hi, inv_temp, pos_dev_or_null,
                                                     ld_tokens, rows, guidance_scale);
  return check_launch("sample_rows_kernel");
}

static int caption_next_launch(cudaStream_t stream, int32_t* tokens, long long ld, const int32_t* prefix,
                               long long ld_prefix, const int32_t* lens, int rows, int text_len, int text_vocab_size,
                               int padding_id, int pad_base, int pos, const int32_t* pos_dev) {
  DB200_REQUIRE(tokens && prefix && lens, DB200_E_INVALID, "caption_next: null pointer");
  DB200_REQUIRE(rows > 0 && text_len >= 1 && ld >= text_len && ld_prefix >= text_len, DB200_E_INVALID,
                "caption_next: rows %d text_len %d ld %lld ld_prefix %lld", rows, text_len, ld, ld_prefix);
  DB200_REQUIRE(text_vocab_size > 0 && padding_id >= 0 && padding_id < text_vocab_size, DB200_E_INVALID,
                "caption_next: padding_id %d outside [0, %d)", padding_id, text_vocab_size);
  DB200_REQUIRE(pad_base < 0 || (pad_base >= text_vocab_size && (long long)pad_base + text_len <= 2147483647LL),
                DB200_E_INVALID, "caption_next: pad_base %d with text_vocab_size %d", pad_base, text_vocab_size);
  DB200_REQUIRE(pos_dev || (pos >= 0 && pos + 1 < text_len), DB200_E_INVALID,
                "caption_next: column %d outside [1, %d)", pos + 1, text_len);
  caption_next_kernel<<<(rows + 127) / 128, 128, 0, stream>>>(tokens, ld, prefix, ld_prefix, lens, rows, text_len,
                                                              text_vocab_size, padding_id, pad_base, pos, pos_dev);
  return check_launch("caption_next_kernel");
}

extern "C" int db200_caption_next(db200_stream_t stream_, int32_t* tokens, long long ld_tokens, const int32_t* prefix,
                                  long long ld_prefix, const int32_t* lens, int rows, int text_len,
                                  int text_vocab_size, int padding_id, int pad_base, int pos) {
  return caption_next_launch(static_cast<cudaStream_t>(stream_), tokens, ld_tokens, prefix, ld_prefix, lens, rows,
                             text_len, text_vocab_size, padding_id, pad_base, pos, nullptr);
}

extern "C" int db200_caption_next_at(db200_stream_t stream_, int32_t* tokens, long long ld_tokens,
                                     const int32_t* prefix, long long ld_prefix, const int32_t* lens, int rows,
                                     int text_len, int text_vocab_size, int padding_id, int pad_base,
                                     const int32_t* pos_dev) {
  DB200_REQUIRE(pos_dev, DB200_E_INVALID, "caption_next_at: null position pointer");
  return caption_next_launch(static_cast<cudaStream_t>(stream_), tokens, ld_tokens, prefix, ld_prefix, lens, rows,
                             text_len, text_vocab_size, padding_id, pad_base, 0, pos_dev);
}

extern "C" int db200_onehot_rows_f32(db200_stream_t stream_, const int32_t* idx, float* y, int rows, int K,
                                     int offset) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(idx && y && rows > 0 && K > 0, DB200_E_INVALID, "onehot_rows: bad argument");
  onehot_rows_kernel<<<rows, 256, 0, stream>>>(idx, y, K, offset);
  return check_launch("onehot_rows_kernel");
}

static unsigned copy_blocks(long long total) {
  const long long want = (total + 255) / 256, cap = (long long)sm_count() * 16;
  return (unsigned)(want < cap ? want : cap);
}

extern "C" int db200_kv_cache_fill(db200_stream_t stream_, const void* qkv, void* k_cache, void* v_cache, int B, int P,
                                   int H, int dh, int S_cache, int rep) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(qkv && k_cache && v_cache, DB200_E_INVALID, "kv_cache_fill: null pointer");
  DB200_REQUIRE(B > 0 && P > 0 && H > 0 && dh > 0 && S_cache > 0 && rep >= 1, DB200_E_INVALID,
                "kv_cache_fill: B %d P %d H %d dh %d S_cache %d rep %d", B, P, H, dh, S_cache, rep);
  DB200_REQUIRE(P <= S_cache, DB200_E_INVALID, "kv_cache_fill: %d prompt positions exceed the cache's %d", P, S_cache);
  DB200_REQUIRE((H * dh) % 8 == 0 && aligned16(qkv) && aligned16(k_cache) && aligned16(v_cache), DB200_E_ALIGN,
                "kv_cache_fill: H*dh %d not a multiple of 8 or unaligned pointer", H * dh);
  const int n16 = H * dh / 8;
  const long long total = (long long)B * P * 2 * n16;
  kv_cache_fill_kernel<<<copy_blocks(total), 256, 0, stream>>>(static_cast<const uint4*>(qkv),
                                                              static_cast<uint4*>(k_cache),
                                                              static_cast<uint4*>(v_cache), P, S_cache, rep, n16, total);
  return check_launch("kv_cache_fill_kernel");
}

extern "C" int db200_rows_repeat(db200_stream_t stream_, const void* src, long long ld_src, void* dst, int B, int d,
                                 int rep) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(src && dst, DB200_E_INVALID, "rows_repeat: null pointer");
  DB200_REQUIRE(B > 0 && d > 0 && rep >= 1 && ld_src >= d, DB200_E_INVALID, "rows_repeat: B %d d %d rep %d ld %lld", B,
                d, rep, ld_src);
  DB200_REQUIRE(d % 8 == 0 && ld_src % 8 == 0 && aligned16(src) && aligned16(dst), DB200_E_ALIGN,
                "rows_repeat: d %d / ld %lld not multiples of 8 or unaligned pointer", d, ld_src);
  const long long total = (long long)B * (d / 8);
  rows_repeat_kernel<<<copy_blocks(total), 256, 0, stream>>>(static_cast<const uint4*>(src), ld_src / 8,
                                                            static_cast<uint4*>(dst), d / 8, rep, total);
  return check_launch("rows_repeat_kernel");
}
