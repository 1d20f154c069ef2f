// Host-side plumbing shared by every translation unit of libdalle_b200.so:
// error codes + thread-local message (the C ABI never throws, never exits), TMA tensor-map encoding via the
// driver entry point (no link-time dependency on libcuda), launch checks.
#pragma once
#include <cmath>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "../../include/dalle_b200.h"

namespace db200 {

typedef __nv_bfloat16 bf16;

// ---- error handling ------------------------------------------------------------------------------
int set_error(int code, const char* fmt, ...);  // stores message in a thread-local buffer, returns code
int check_launch(const char* what);             // cudaGetLastError() -> DB200_E_CUDA

#define DB200_REQUIRE(cond, code, ...)                   \
  do {                                                   \
    if (!(cond)) return ::db200::set_error((code), __VA_ARGS__); \
  } while (0)

#define DB200_CUDA(call)                                                                               \
  do {                                                                                                 \
    cudaError_t e__ = (call);                                                                          \
    if (e__ != cudaSuccess)                                                                            \
      return ::db200::set_error(DB200_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), \
                                __FILE__, __LINE__);                                                   \
  } while (0)

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// the weighted cross-entropy descriptor (db200_gemm_bf16_ce_weighted, db200_ce_finish_weighted)
static inline int ce_weights_check(const db200_ce_weights* w, const char* what) {
  DB200_REQUIRE(w != nullptr, DB200_E_INVALID, "%s: NULL weights descriptor", what);
  DB200_REQUIRE(w->period > 0 && w->text_rows >= 0 && w->text_rows <= w->period, DB200_E_INVALID,
                "%s: need period > 0 and 0 <= text_rows <= period (got %d, %d)", what, w->period, w->text_rows);
  DB200_REQUIRE(std::isfinite(w->a_text) && std::isfinite(w->a_image) && std::isfinite(w->z_loss) && w->a_text >= 0.f &&
                    w->a_image >= 0.f && w->z_loss >= 0.f,
                DB200_E_INVALID, "%s: a_text, a_image and z_loss must be finite and >= 0", what);
  return DB200_OK;
}

// ---- TMA tensor maps ------------------------------------------------------------------------------
// rank <= 5; dims[0] is the innermost (contiguous) dimension; strides_bytes[i] is the byte stride of dims[i+1].
// All maps use bf16 elements, 128-byte swizzle, zero OOB fill.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box);

static inline int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t ld_elems,
                               uint32_t box_inner, uint32_t box_outer) {
  uint64_t dims[2] = {inner, outer};
  uint64_t strides[1] = {ld_elems * 2};
  uint32_t box[2] = {box_inner, box_outer};
  return make_tmap_bf16(out, base, 2, dims, strides, box);
}

int sm_count();  // cached cudaDevAttrMultiProcessorCount of the current device

// ---- order-fixed reductions ------------------------------------------------------------------------
// Sums that many CTAs contribute to are not accumulated with float atomics (their order, and so the rounding, would
// change from run to run): every CTA stores its partial into a workspace the caller passes in, and one reduction kernel
// adds the partials in a fixed order on the same stream.
// true if the caller's workspace holds `need` bytes and is 16-byte aligned
static inline bool workspace_ok(const void* ws, int64_t bytes, int64_t need) {
  return need <= 0 || (ws != nullptr && bytes >= need && aligned16(ws));
}
// dst[c] += sum over r = 0, 1, ... rows-1 of ws[r * cols + c]
int reduce_rows_add(cudaStream_t stream, const float* ws, int rows, int cols, float* dst);
// D[m * ldd + n] += sum over s = 0 .. splits-1 of ws[(s * M + m) * N + n]
int reduce_splits_add(cudaStream_t stream, const float* ws, int splits, int M, int N, float* D, long long ldd);

}  // namespace db200
