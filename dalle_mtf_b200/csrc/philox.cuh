// Counter-based dropout masks: Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11)
// and the two index layouts every dropout site of the DALL-E step uses.
//
// A keep decision is a pure function of (seed, step, site, global element index), so the forward, a recomputed
// forward and the backward draw the same mask without storing it, and the mask of a row does not depend on which rank
// or micro-batch holds that row.
//   key     = (lo32(seed), hi32(seed))
//   counter = (lo32(n), hi32(n), site, step); the element reads word w of the four output words
//   elementwise [rows][cols] tensor whose row 0 is global row row0:  e = (row0 + r) * cols + c,  n = e >> 2,  w = e & 3
//   attention weights (b, h, i, j), b global, S2 = ceil(S / 2):      n = ((b H + h) S2 + i/2) S2 + j/2,
//                                                                    w = 2 (i & 1) + (j & 1)
//   keep iff word >= threshold (threshold = floor(rate * 2^32)); kept values are multiplied by scale = 1 / (1 - rate)
#pragma once
#include "common.cuh"

namespace db200 {

#if defined(__CUDACC__)
#define DB200_HD __host__ __device__ __forceinline__
#else
#define DB200_HD inline
#endif

DB200_HD void philox_mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
#if defined(__CUDA_ARCH__)
  hi = __umulhi(a, b);
  lo = a * b;
#else
  const uint64_t p = (uint64_t)a * b;
  hi = (uint32_t)(p >> 32);
  lo = (uint32_t)p;
#endif
}

// Philox4x32 with 10 rounds: the round function and key schedule of Random123 (and of curand_Philox4x32_10)
DB200_HD uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    uint32_t hi0, lo0, hi1, lo1;
    philox_mulhilo(0xD2511F53u, c.x, hi0, lo0);
    philox_mulhilo(0xCD9E8D57u, c.z, hi1, lo1);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// the four words of block n of a site
DB200_HD uint4 dropout_block(const db200_dropout& d, uint64_t n) {
  return philox4x32_10(make_uint4((uint32_t)n, (uint32_t)(n >> 32), d.site, d.step), (uint32_t)d.seed,
                       (uint32_t)(d.seed >> 32));
}

// multiplier of one word: scale if kept, 0 if dropped
DB200_HD float dropout_mul(const db200_dropout& d, uint32_t word) { return word >= d.threshold ? d.scale : 0.f; }

// elementwise layout: block index of the 4 elements starting at column c (c % 4 == 0, cols % 4 == 0) of local row r
DB200_HD uint64_t dropout_elem_block(const db200_dropout& d, long long r, long long cols, long long c) {
  return (uint64_t)((d.row0 + r) * cols + c) >> 2;
}

// attention layout: block of (b, h, i, j) with b the LOCAL sequence index (d.row0 is the first global sequence)
DB200_HD uint64_t dropout_attn_block(const db200_dropout& d, int b, int h, int H, int S2, int i, int j) {
  return (((uint64_t)(d.row0 + b) * H + h) * S2 + (i >> 1)) * S2 + (j >> 1);
}

DB200_HD uint32_t uint4_word(const uint4& v, int w) {
  return w == 0 ? v.x : (w == 1 ? v.y : (w == 2 ? v.z : v.w));
}

// `d` is active (non-NULL with a non-zero drop probability)
inline bool dropout_active(const db200_dropout* d) { return d != nullptr && d->threshold != 0; }

}  // namespace db200
