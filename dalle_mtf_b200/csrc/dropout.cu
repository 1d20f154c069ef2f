// D0 — materialised dropout masks (tests and oracle comparisons): the keep bits the fused kernels regenerate, from the
// same device functions (philox.cuh).
#include "common.cuh"
#include "philox.cuh"

namespace db200 {

__global__ void dropout_mask_elem_kernel(const db200_dropout dr, long long rows, long long cols,
                                         uint8_t* __restrict__ keep) {
  const long long total = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols, c = i - r * cols;
    const uint64_t e = (uint64_t)((dr.row0 + r) * cols + c);
    keep[i] = uint4_word(dropout_block(dr, e >> 2), (int)(e & 3)) >= dr.threshold;
  }
}

__global__ void dropout_mask_attn_kernel(const db200_dropout dr, int B, int H, int S, uint8_t* __restrict__ keep) {
  const long long total = (long long)B * H * S * S;
  const int S2 = (S + 1) >> 1;
  for (long long x = blockIdx.x * (long long)blockDim.x + threadIdx.x; x < total;
       x += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(x % S);
    const int i = (int)((x / S) % S);
    const long long bh = x / ((long long)S * S);
    const int h = (int)(bh % H), b = (int)(bh / H);
    const uint4 r = dropout_block(dr, dropout_attn_block(dr, b, h, H, S2, i, j));
    keep[x] = uint4_word(r, 2 * (i & 1) + (j & 1)) >= dr.threshold;
  }
}

}  // namespace db200

using namespace db200;

extern "C" int db200_dropout_mask(db200_stream_t stream_, const db200_dropout* d, int layout, int64_t dim0,
                                  int64_t dim1, int64_t dim2, uint8_t* keep) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(d && keep, DB200_E_INVALID, "dropout_mask: NULL descriptor or output");
  DB200_REQUIRE(d->row0 >= 0, DB200_E_INVALID, "dropout_mask: row0 must be >= 0");
  long long total;
  if (layout == DB200_DROPOUT_ELEMENTWISE) {
    DB200_REQUIRE(dim0 > 0 && dim1 > 0, DB200_E_INVALID, "dropout_mask: rows, cols must be positive");
    total = dim0 * dim1;
  } else if (layout == DB200_DROPOUT_ATTENTION) {
    DB200_REQUIRE(dim0 > 0 && dim1 > 0 && dim2 > 0 && dim2 <= INT32_MAX && dim0 * dim1 <= INT32_MAX, DB200_E_INVALID,
                  "dropout_mask: B, H, S must be positive");
    total = dim0 * dim1 * dim2 * dim2;
  } else {
    return set_error(DB200_E_INVALID, "dropout_mask: unknown layout %d", layout);
  }
  const long long want = (total + 255) / 256;
  const int blocks = (int)(want < sm_count() * 16 ? want : sm_count() * 16);
  if (layout == DB200_DROPOUT_ELEMENTWISE)
    dropout_mask_elem_kernel<<<blocks, 256, 0, stream>>>(*d, dim0, dim1, keep);
  else
    dropout_mask_attn_kernel<<<blocks, 256, 0, stream>>>(*d, (int)dim0, (int)dim1, (int)dim2, keep);
  return check_launch("dropout_mask_kernel");
}
