// Token shift (extension; DALLE-pytorch's PreShiftToken) on the LayerNorm outputs a q|k|v or W1 product reads.
//
// A row of y is d bf16 values of one position p; c = d / 4.  The first quarter [0, c) of position p is replaced by
// the same quarter of its source position for the "top" chunk, the second quarter [c, 2c) by that of the "left"
// chunk's source, and [2c, d) is kept:
//   text p < TL      : both chunks from p - 1 (zeros at p = 0)
//   image (r, k)     : [0, c) from p - W if r >= 1, [c, 2c) from p - 1 if k >= 1, zeros otherwise
// (u = p - TL, r = u / W, k = u % W).  Text never reads image and image never reads text.  Pure data movement: the
// result is exact.  d % 32 == 0 makes c a whole number of 16-byte vectors, so every kernel copies uint4 vectors.
#include <climits>

#include "common.cuh"

namespace db200 {

// The position whose chunk ch (0 top, 1 left) position p reads, or -1 for zeros.
__device__ __forceinline__ int shift_src(int p, int ch, int TL, int W) {
  if (p < TL) return p - 1;
  const int u = p - TL;
  if (ch == 0) return u >= W ? p - W : -1;
  return u % W ? p - 1 : -1;
}

// The transpose: the position whose chunk ch reads position p, or -1; n is the sequence length.
__device__ __forceinline__ int shift_dst(int p, int ch, int TL, int W, int n) {
  int q;
  if (p < TL) {
    q = p + 1 < TL ? p + 1 : -1;
  } else {
    const int u = p - TL;
    if (ch == 0) q = u + W < W * W ? p + W : -1;
    else         q = u % W + 1 < W ? p + 1 : -1;
  }
  return q < n ? q : -1;
}

// out = shift(in) (BWD: shift^T(in)), row t at position t mod S; nv = d / 8 vectors per row, cv = c / 8.
template <bool BWD>
__global__ void __launch_bounds__(256)
shift_tokens_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, long long total, int nv, int cv, int S,
                    int TL, int W) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / nv;
    const int v = (int)(i - t * nv);
    uint4 val = make_uint4(0u, 0u, 0u, 0u);
    if (v >= 2 * cv) {
      val = in[i];
    } else {
      const int p = (int)(t % S);
      const int q = BWD ? shift_dst(p, v >= cv, TL, W, S) : shift_src(p, v >= cv, TL, W);
      if (q >= 0) val = in[i + (long long)(q - p) * nv];
    }
    out[i] = val;
  }
}

// One decoding step at position p = *pos_dev (or pos) for every row b: cache[b][p] = y[b][0, 2c), then y[b][0, 2c)
// = the shifted chunks read from cache[b] (positions < p, written by earlier steps or the prefill).  hv = 2 cv
// vectors per cache position.  A position outside [0, S) leaves y and the cache unchanged.
__global__ void __launch_bounds__(256)
shift_decode_kernel(uint4* __restrict__ y, uint4* __restrict__ cache, int rows, int nv, int cv, int S, int TL, int W,
                    int pos, const int* __restrict__ pos_dev) {
  const int p = pos_dev ? *pos_dev : pos;
  if (p < 0 || p >= S) return;
  const int hv = 2 * cv;
  const long long total = (long long)rows * hv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / hv;
    const int v = (int)(i - b * hv);
    uint4* row = cache + b * S * hv;
    uint4* yv = y + b * nv + v;
    row[(long long)p * hv + v] = *yv;
    const int q = shift_src(p, v >= cv, TL, W);
    *yv = q >= 0 ? row[(long long)q * hv + v] : make_uint4(0u, 0u, 0u, 0u);
  }
}

// Prefill hand-off: cache[b * rep + r][p] = y[b * P + p][0, 2c) for p < P, r < rep.
__global__ void __launch_bounds__(256)
shift_cache_fill_kernel(const uint4* __restrict__ y, uint4* __restrict__ cache, int P, int S, int rep, int nv, int hv,
                        long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / hv;
    const int v = (int)(i - t * hv);
    const int p = (int)(t % P);
    const long long b = t / P;
    const uint4 val = y[t * nv + v];
    for (int r = 0; r < rep; ++r) cache[((b * rep + r) * S + p) * hv + v] = val;
  }
}

static int shift_grid(long long work) {
  const long long cap = (long long)sm_count() * 16;
  const long long blocks = (work + 255) / 256;
  return (int)(blocks < 1 ? 1 : (blocks < cap ? blocks : cap));
}

// Checks shared by the shift entry points: S positions of a TL + W^2 sequence, d % 32 == 0.
static int shift_geometry(int rows, int S, int d, int TL, int W, const char* what) {
  DB200_REQUIRE(rows > 0 && S > 0 && d > 0 && TL >= 0 && W > 0, DB200_E_INVALID,
                "%s: need rows, S, d, grid_w > 0 and text_len >= 0 (got rows=%d S=%d d=%d text_len=%d grid_w=%d)",
                what, rows, S, d, TL, W);
  DB200_REQUIRE(d % 32 == 0, DB200_E_INVALID, "%s: d %d is not a multiple of 32", what, d);
  DB200_REQUIRE((long long)TL + (long long)W * W <= INT_MAX && S <= TL + W * W, DB200_E_INVALID,
                "%s: S %d exceeds text_len %d + grid_w^2 (grid_w %d)", what, S, TL, W);
  return 0;
}

// Whether the byte ranges [a, a + na) and [b, b + nb) share a byte.
static bool overlaps(const void* a, long long na, const void* b, long long nb) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return x < y + (uintptr_t)nb && y < x + (uintptr_t)na;
}

static int shift_launch(cudaStream_t stream, const void* in, void* out, int rows, int S, int d, int TL, int W, bool bwd,
                        const char* what) {
  DB200_REQUIRE(in && out, DB200_E_INVALID, "%s: NULL pointer", what);
  const int err = shift_geometry(rows, S, d, TL, W, what);
  if (err) return err;
  const long long bytes = (long long)rows * d * 2;
  DB200_REQUIRE(!overlaps(in, bytes, out, bytes), DB200_E_INVALID, "%s: input and output overlap", what);
  DB200_REQUIRE(aligned16(in) && aligned16(out), DB200_E_ALIGN, "%s: pointers must be 16-byte aligned", what);
  const int nv = d / 8;
  const long long total = (long long)rows * nv;
  const uint4* src = static_cast<const uint4*>(in);
  uint4* dst = static_cast<uint4*>(out);
  if (bwd) shift_tokens_kernel<true><<<shift_grid(total), 256, 0, stream>>>(src, dst, total, nv, nv / 4, S, TL, W);
  else     shift_tokens_kernel<false><<<shift_grid(total), 256, 0, stream>>>(src, dst, total, nv, nv / 4, S, TL, W);
  return check_launch(what);
}

static int shift_decode_launch(cudaStream_t stream, void* y, void* cache, int rows, int S, int d, int TL, int W,
                               int pos, const int32_t* pos_dev, const char* what) {
  DB200_REQUIRE(y && cache, DB200_E_INVALID, "%s: NULL pointer", what);
  const int err = shift_geometry(rows, S, d, TL, W, what);
  if (err) return err;
  DB200_REQUIRE(!overlaps(y, (long long)rows * d * 2, cache, (long long)rows * S * d), DB200_E_INVALID,
                "%s: rows and cache overlap", what);
  DB200_REQUIRE(aligned16(y) && aligned16(cache), DB200_E_ALIGN, "%s: pointers must be 16-byte aligned", what);
  const int nv = d / 8;
  shift_decode_kernel<<<shift_grid((long long)rows * (nv / 2)), 256, 0, stream>>>(
      static_cast<uint4*>(y), static_cast<uint4*>(cache), rows, nv, nv / 4, S, TL, W, pos, pos_dev);
  return check_launch(what);
}

}  // namespace db200

using namespace db200;

extern "C" int db200_shift_tokens_fwd(db200_stream_t stream, const void* y_bf16, void* out_bf16, int rows, int S, int d,
                                      int text_len, int grid_w) {
  return shift_launch(reinterpret_cast<cudaStream_t>(stream), y_bf16, out_bf16, rows, S, d, text_len, grid_w, false,
                      "shift_tokens_fwd");
}

extern "C" int db200_shift_tokens_bwd(db200_stream_t stream, const void* dout_bf16, void* dy_bf16, int rows, int S,
                                      int d, int text_len, int grid_w) {
  return shift_launch(reinterpret_cast<cudaStream_t>(stream), dout_bf16, dy_bf16, rows, S, d, text_len, grid_w, true,
                      "shift_tokens_bwd");
}

extern "C" int db200_shift_tokens_decode(db200_stream_t stream, void* y_bf16, void* cache_bf16, int rows, int S, int d,
                                         int text_len, int grid_w, int pos) {
  DB200_REQUIRE(pos >= 0 && pos < S, DB200_E_INVALID, "shift_tokens_decode: position %d outside [0, %d)", pos, S);
  return shift_decode_launch(reinterpret_cast<cudaStream_t>(stream), y_bf16, cache_bf16, rows, S, d, text_len, grid_w,
                             pos, nullptr, "shift_tokens_decode");
}

extern "C" int db200_shift_tokens_decode_dev(db200_stream_t stream, void* y_bf16, void* cache_bf16, int rows, int S,
                                             int d, int text_len, int grid_w, const int32_t* pos_dev) {
  DB200_REQUIRE(pos_dev, DB200_E_INVALID, "shift_tokens_decode_dev: NULL pos_dev");
  return shift_decode_launch(reinterpret_cast<cudaStream_t>(stream), y_bf16, cache_bf16, rows, S, d, text_len, grid_w,
                             -1, pos_dev, "shift_tokens_decode_dev");
}

extern "C" int db200_shift_cache_fill(db200_stream_t stream, const void* y_bf16, void* cache_bf16, int B, int P, int d,
                                      int S_cache, int rep) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  DB200_REQUIRE(y_bf16 && cache_bf16, DB200_E_INVALID, "shift_cache_fill: NULL pointer");
  DB200_REQUIRE(B > 0 && P > 0 && d > 0 && S_cache > 0 && rep >= 1, DB200_E_INVALID,
                "shift_cache_fill: B %d P %d d %d S_cache %d rep %d", B, P, d, S_cache, rep);
  DB200_REQUIRE(d % 32 == 0, DB200_E_INVALID, "shift_cache_fill: d %d is not a multiple of 32", d);
  DB200_REQUIRE(P <= S_cache, DB200_E_INVALID, "shift_cache_fill: %d prompt positions exceed the cache's %d", P,
                S_cache);
  DB200_REQUIRE(!overlaps(y_bf16, (long long)B * P * d * 2, cache_bf16, (long long)B * rep * S_cache * d),
                DB200_E_INVALID,
                "shift_cache_fill: rows and cache overlap");
  DB200_REQUIRE(aligned16(y_bf16) && aligned16(cache_bf16), DB200_E_ALIGN,
                "shift_cache_fill: pointers must be 16-byte aligned");
  const int nv = d / 8, hv = nv / 2;
  const long long total = (long long)B * P * hv;
  shift_cache_fill_kernel<<<shift_grid(total), 256, 0, s>>>(static_cast<const uint4*>(y_bf16),
                                                            static_cast<uint4*>(cache_bf16), P, S_cache, rep, nv, hv,
                                                            total);
  return check_launch("shift_cache_fill");
}
