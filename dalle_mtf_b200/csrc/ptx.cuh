// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma operand descriptors.
// Everything here is device-side and header-only.  No CUTLASS/CuTe dependency.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

namespace db200 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a dead-locked pipeline traps (-> launch error) instead of hanging the GPU box.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3ff) == 0 && clock64() - t0 > 4000000000ll) {  // ~2 s at 2 GHz
      printf("db200: mbarrier wait timeout block=%d thread=%d bar=0x%x parity=%u\n", blockIdx.x, threadIdx.x, bar,
             parity);
      __trap();
    }
  }
}

// Same bound without the report, for waits inside a wgmma pipeline: a printf call there makes ptxas serialise the
// warpgroup MMAs of the whole kernel.
__device__ __forceinline__ void mbar_wait_mma(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity))
    if ((++spins & 0x3ff) == 0 && clock64() - t0 > 4000000000ll) __trap();
}

// generic-proxy writes (st.shared) -> visible to the async proxy (TMA store / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA loads (tile mode), completion on an mbarrier (complete_tx::bytes)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          dst),
      "l"(m), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];" ::"r"(dst),
      "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(dst),
      "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], "
      "[%2];" ::"r"(dst),
      "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
// L2 prefetch of a 4-D box (no smem destination, no barrier): hides the DRAM part of a later TMA load's latency
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* m, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];" ::"l"(m), "r"(c0), "r"(c1),
               "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(m), "r"(src),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read0() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// elect.sync: true in exactly one (the lowest active) lane of a converged warp.  ptxas recognises the pattern and emits a
// single ELECT + predicated / uniformly-branched code for the guarded block — unlike `lane == 0`, which it must treat as
// an arbitrary per-thread predicate (a lane-by-lane "waterfall" loop around every uniform-datapath instruction).
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred)
      :
      : "memory");
  return pred != 0;
}

// setmaxnreg: change the calling warpgroup's per-thread register count (every warp of the warpgroup executes it;
// R is a multiple of 8 in [24, 256]).  dec returns registers to the CTA's pool, inc waits until the pool can supply them.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}

// ----------------------------------------------------------------------------------------------
// wgmma shared-memory operand descriptor (PTX ISA "Matrix Descriptor Format" for wgmma), 128-byte swizzle.
//   K-major tile  [rows][64 bf16]        : rows are 128 B apart, 8-row groups SBO=1024 B apart, LBO unused.
//   MN-major slab [k rows][64 bf16 of MN]: k rows 128 B apart, 8-k groups SBO=1024 B apart,
//                                          64-wide MN atoms LBO bytes apart.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);             // [0,14)  start address >> 4
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;     // [16,30) leading byte offset >> 4
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;     // [32,46) stride byte offset >> 4
  d |= 1ull << 62;                                                   // [62,64) layout type 1 = SWIZZLE_128B
  return d;
}

// Byte offset of element (row, col) inside a [rows][64 bf16] tile stored with the 128-byte swizzle that TMA
// (CU_TENSOR_MAP_SWIZZLE_128B) and the wgmma SW128 descriptor agree on: 16-byte chunk index XOR (row % 8).
__device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t col) {
  return row * 128u + ((((col >> 3) ^ (row & 7u)) & 7u) << 4) + ((col & 7u) << 1);
}

// ----------------------------------------------------------------------------------------------
// small numeric helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace db200
