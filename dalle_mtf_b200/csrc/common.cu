#include "common.cuh"

#include <cstring>
#include <mutex>

namespace db200 {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

static unsigned long long g_launches = 0;  // kernels launched through this library (bench.py reports the delta)

int check_launch(const char* what) {
  __atomic_fetch_add(&g_launches, 1ull, __ATOMIC_RELAXED);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(DB200_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return DB200_OK;
}

typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_tiled_fn get_encode_fn() {
  static encode_tiled_fn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<encode_tiled_fn>(p);
  });
  return fn;
}

// cuTensorMapEncodeTiled costs a microsecond or two of host time per call and every GEMM / conv / attention launch
// needs two to four maps.  A map depends only on (base pointer, geometry), and the engines launch the same kernels on
// the same pre-allocated buffers every step, so encoded maps are cached (per thread; dropped wholesale when full).
struct TmapKey {
  uint64_t v[16];
  bool operator==(const TmapKey& o) const { return memcmp(v, o.v, sizeof(v)) == 0; }
};
struct TmapEntry {
  TmapKey key;
  CUtensorMap map;
  bool used = false;
};
static constexpr int TMAP_CACHE = 2048;  // power of two

static int make_tmap_bf16_uncached(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                                   const uint64_t* strides_bytes, const uint32_t* box);

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box) {
  static thread_local TmapEntry* cache = new TmapEntry[TMAP_CACHE];
  TmapKey k;
  memset(&k, 0, sizeof(k));
  k.v[0] = reinterpret_cast<uint64_t>(base);
  k.v[1] = (uint64_t)rank;
  for (int i = 0; i < rank && i < 5; ++i) { k.v[2 + i] = dims[i]; k.v[11 + i] = box[i]; }
  for (int i = 0; i + 1 < rank && i < 4; ++i) k.v[7 + i] = strides_bytes[i];
  uint64_t h = 1469598103934665603ull;
  for (int i = 0; i < 16; ++i) { h ^= k.v[i]; h *= 1099511628211ull; }
  TmapEntry& e = cache[(h ^ (h >> 29)) & (TMAP_CACHE - 1)];
  if (e.used && e.key == k) {
    *out = e.map;
    return DB200_OK;
  }
  const int rc = make_tmap_bf16_uncached(out, base, rank, dims, strides_bytes, box);
  if (rc == DB200_OK) { e.key = k; e.map = *out; e.used = true; }
  return rc;
}

static int make_tmap_bf16_uncached(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                                   const uint64_t* strides_bytes, const uint32_t* box) {
  encode_tiled_fn fn = get_encode_fn();
  if (!fn) return set_error(DB200_E_CUDA, "cuTensorMapEncodeTiled driver entry point not available");
  if (!aligned16(base)) return set_error(DB200_E_ALIGN, "TMA base pointer %p is not 16-byte aligned", base);
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (box[i] == 0 || box[i] > 256) return set_error(DB200_E_INVALID, "TMA box dim %d = %u out of range", i, box[i]);
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    if (strides_bytes[i] % 16 != 0)
      return set_error(DB200_E_ALIGN, "TMA stride %d = %llu bytes is not a multiple of 16", i,
                       (unsigned long long)strides_bytes[i]);
  }
  if (box[0] * 2 > 128) return set_error(DB200_E_INVALID, "TMA inner box exceeds the 128-byte swizzle span");
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(DB200_E_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return DB200_OK;
}

// block = 32 columns x 8 row lanes: lane k sums rows k, k + 8, ... in order, then the 8 lane sums are added in lane order
__global__ void __launch_bounds__(256)
reduce_rows_add_kernel(const float* __restrict__ ws, int rows, int cols, float* __restrict__ dst) {
  __shared__ float part[8][32];
  const int cx = threadIdx.x & 31, k = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  float s = 0.f;
  if (c < cols)
    for (int r = k; r < rows; r += 8) s += ws[(long long)r * cols + c];
  part[k][cx] = s;
  __syncthreads();
  if (k == 0 && c < cols) {
    float t = part[0][cx];
#pragma unroll
    for (int j = 1; j < 8; ++j) t += part[j][cx];
    dst[c] += t;
  }
}

__global__ void reduce_splits_add_kernel(const float* __restrict__ ws, int splits, int M, int N, float* __restrict__ D,
                                         long long ldd) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long mn = (long long)M * N;
  if (i >= mn) return;
  float s = 0.f;
  for (int k = 0; k < splits; ++k) s += ws[k * mn + i];
  const long long m = i / N, n = i - m * N;
  D[m * ldd + n] += s;
}

int reduce_rows_add(cudaStream_t stream, const float* ws, int rows, int cols, float* dst) {
  reduce_rows_add_kernel<<<(cols + 31) / 32, 256, 0, stream>>>(ws, rows, cols, dst);
  return check_launch("reduce_rows_add_kernel");
}

int reduce_splits_add(cudaStream_t stream, const float* ws, int splits, int M, int N, float* D, long long ldd) {
  const long long mn = (long long)M * N;
  reduce_splits_add_kernel<<<(unsigned)((mn + 255) / 256), 256, 0, stream>>>(ws, splits, M, N, D, ldd);
  return check_launch("reduce_splits_add_kernel");
}

int g_reserved_sms = 0;   // SMs left to a concurrently running collective (set once at start-up)

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = n > 0 ? n : 132;
  }
  const int n = cached[dev] - g_reserved_sms;
  return n > 16 ? n : 16;
}

}  // namespace db200

extern "C" {

const char* db200_last_error(void) { return db200::g_err; }
int db200_version(void) { return 100; }
unsigned long long db200_launch_count(void) { return __atomic_load_n(&db200::g_launches, __ATOMIC_RELAXED); }

int db200_device_check(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return db200::set_error(DB200_E_CUDA, "cudaGetDevice: %s", cudaGetErrorString(e));
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0)
    return db200::set_error(DB200_E_UNSUPPORTED, "device %d is sm_%d%d; libdalle_b200 ships sm_90a code only", dev,
                            major, minor);
  return DB200_OK;
}
}

// The persistent kernels (GEMM, convolutions) launch one CTA per SM that needs the whole SM (shared memory,
// registers): a collective whose CTAs occupy k SMs while they run would push k of those CTAs into a second wave.
// With k SMs reserved the grids are sized to sm_count - k and both fit side by side (data-parallel runs reserve the
// CTA cap of the overlapped communicator).
extern "C" int db200_set_reserved_sms(int n) {
  if (n < 0 || n > 64) return db200::set_error(DB200_E_INVALID, "set_reserved_sms: %d not in [0, 64]", n);
  db200::g_reserved_sms = n;
  return DB200_OK;
}
