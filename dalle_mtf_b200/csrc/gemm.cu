// K3/K5/K6/K7/K8 — persistent, warp-specialised bf16 GEMM on wgmma for sm_90a.
//
//   D[M,N] = A[M,K] * B[K,N],  fp32 accumulation in registers, operands staged in shared memory by TMA (128B swizzle).
//
//   warp 0     : TMA producer (one elected lane)            smem ring: STAGES x {A 128x64, B BNx64} bf16
//   warps 1-3  : idle (they hand their registers to the other warpgroups and exit)
//   warps 4-11 : two MMA warpgroups.  Warpgroup g issues wgmma m64 x BN x 16 for rows [64g, 64g+64) of the tile and at
//                the end of the tile writes its accumulators to a shared-memory accumulator tile.
//   warps 12-15: the epilogue warpgroup.  Warp e owns rows [32e, 32e+32) of the accumulator tile, one row per thread,
//                and runs the epilogue on it half tile by half tile -> bias / ReLU / GELU / residual / split-K
//                reduction / cross-entropy statistics and gradient.
//
// The accumulator tile is single-buffered and handed over through two named barriers (FULL: written by the MMA
// warpgroups; EMPTY: read by the epilogue).  The MMA warpgroups run the next tile's mainloop while the epilogue works
// on the previous one, and wait for EMPTY only before their next store; the producer keeps loading throughout.
//
// Either operand may be K-major or MN-major in global memory; the tensor maps and the wgmma descriptors absorb the
// difference, so forward (x*W), dgrad (dy*W^T) and wgrad (x^T*dy) are the same kernel.
//
// Reference call sites replaced: every mtf einsum / mtf.layers.dense of src/dalle_mtf/models.py (235-244, 303-311,
// 317-324, 361-371, 391-395) and their gradients produced by mtf.gradients (src/optimizers.py:34).
#include "gemm_common.cuh"
#include "wgmma.cuh"

namespace db200 {

// BN = 128: the 128 x 128 fp32 accumulator tile (64 KiB), four 32 KiB stages and the epilogue warps' staging blocks fit
// the 227 KiB of an H100 SM; a second accumulator tile or a fifth stage does not.
constexpr int GBN = 128;
constexpr int G_STAGES = 4;
constexpr uint32_t G_B_BYTES = GBN * BK * 2;
constexpr uint32_t G_STAGE_BYTES = A_BYTES + G_B_BYTES;
constexpr uint32_t G_ACC_BYTES = BM * GBN * 4;
constexpr size_t G_SMEM_BYTES =
    1024 /*align slack*/ + G_ACC_BYTES + size_t(G_STAGES) * G_STAGE_BYTES + 256 /*barriers*/ + 4 * STG_BYTES;
static_assert(G_SMEM_BYTES <= 227 * 1024, "GEMM shared memory exceeds the H100 per-block limit");

// 512 threads compile to 128 registers each; setmaxnreg moves the producer warpgroup's share to the MMA warpgroups
// (64 accumulators + the mainloop) and the epilogue (two 32-column accumulator chunks + the output chunk in flight).
constexpr int G_REGS_PRODUCER = 40, G_REGS_MMA = 152, G_REGS_EPI = 168;
static_assert(128 * G_REGS_PRODUCER + 256 * G_REGS_MMA + 128 * G_REGS_EPI <= 65536, "GEMM register budget");
// named barriers of the accumulator-tile hand-off: 256 MMA threads + 128 epilogue threads
constexpr int G_BAR_FULL = 1, G_BAR_EMPTY = 2, G_BAR_HANDOFF_THREADS = 384;

// operand majors (1 = MN-major), compile-time for wgmma; DROP: dropout in the STORE epilogue; WCE: the weighted CE_GRAD
// epilogue (instantiated for the vocabulary product only: A K-major, B MN-major); MLP: the GELU MLP's epilogues,
// G_GELU_FWD (the W1 forward: A K-major, B MN-major) or G_GELU_BWD (its dgrad: both K-major), or the gated MLP's,
// G_GLU_*_FWD (the W1 forward, whose B operand is the [K][2N] value | gate weight) or G_GLU_*_BWD (its dgrad)
constexpr int G_GELU_FWD = 1, G_GELU_BWD = 2;
constexpr int G_GLU_RELU_FWD = 3, G_GLU_GELU_FWD = 4, G_GLU_RELU_BWD = 5, G_GLU_GELU_BWD = 6;
__host__ __device__ constexpr bool glu_fwd(int mlp) { return mlp == G_GLU_RELU_FWD || mlp == G_GLU_GELU_FWD; }
__host__ __device__ constexpr bool glu_bwd(int mlp) { return mlp == G_GLU_RELU_BWD || mlp == G_GLU_GELU_BWD; }
template <int TA, int TB, bool DROP, bool WCE = false, int MLP = 0>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  constexpr int BN = GBN;
  constexpr int STAGES = G_STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;  // SWIZZLE_128B tiles need 1024-byte alignment
  const uint32_t sAcc = base;
  const uint32_t sA = base + G_ACC_BYTES;
  const uint32_t sB = sA + STAGES * A_BYTES;
  const uint32_t bars = sA + STAGES * G_STAGE_BYTES;
  const uint32_t full_bar = bars;                   // STAGES x 8 B
  const uint32_t empty_bar = bars + 8 * STAGES;     // STAGES x 8 B
  const uint32_t stg_base = bars + 256;             // 4 x STG_BYTES, 16-byte aligned

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(full_bar + 8 * i, 1);
      mbar_init(empty_bar + 8 * i, 2);  // one arrive per MMA warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int total_tiles = p.m_tiles * p.n_tiles * p.splits;

  if (warp < 4) {
    setmaxnreg_dec<G_REGS_PRODUCER>();
    if (warp != 0) return;
    // ------------------------------------------------------------------ TMA producer
    // converged warp, issuer picked by elect.sync: TMA instructions compile to plain uniform-datapath code
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      // a GLU forward tile covers 64 output columns: its value slab at n0 and its gate slab at N + n0
      const int m0 = t.m_blk * BM, n0 = t.n_blk * (glu_fwd(MLP) ? 64 : BN);
      for (int kb = t.kb0; kb < t.kb1; ++kb) {
        mbar_wait_mma(empty_bar + 8 * stage, phase ^ 1);
        const uint32_t fb = full_bar + 8 * stage;
        if (elect_one_sync()) {
          mbar_expect_tx(fb, G_STAGE_BYTES);
          const int k0 = kb * BK;
          const uint32_t a_dst = sA + stage * A_BYTES;
          const uint32_t b_dst = sB + stage * G_B_BYTES;
          if (p.a_3d) {
            tma_load_3d(a_dst, &tmA, fb, 0, k0, m0 >> 6);
          } else if (p.a_mn) {
#pragma unroll
            for (int s = 0; s < BM / 64; ++s) tma_load_2d(a_dst + s * SLAB_BYTES, &tmA, fb, m0 + 64 * s, k0);
          } else {
            tma_load_2d(a_dst, &tmA, fb, k0, m0);
          }
          if constexpr (glu_fwd(MLP)) {  // the 2D map of B spans all 2N columns
            tma_load_2d(b_dst, &tmB, fb, n0, k0);
            tma_load_2d(b_dst + SLAB_BYTES, &tmB, fb, p.N + n0, k0);
          } else if (p.b_3d) {
            tma_load_3d(b_dst, &tmB, fb, 0, k0, n0 >> 6);
          } else if (p.b_mn) {
#pragma unroll
            for (int s = 0; s < BN / 64; ++s) tma_load_2d(b_dst + s * SLAB_BYTES, &tmB, fb, n0 + 64 * s, k0);
          } else {
            tma_load_2d(b_dst, &tmB, fb, k0, n0);
          }
        }
        __syncwarp();
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp < 12) {
    // ------------------------------------------------------------------ MMA warpgroups
    setmaxnreg_inc<G_REGS_MMA>();
    const int wg = (warp - 4) >> 2;  // accumulator rows [64 wg, 64 wg + 64)
    // K-major: a K-step advances 16 elements (32 B) inside the 128 B swizzle row and warpgroup g starts 64 rows (8 KiB)
    // in; MN-major: a K-step is 16 k-rows (2 KiB) and warpgroup g takes the g-th 64-wide slab (SLAB_BYTES apart).
    constexpr uint64_t astep = TA ? 128u : 2u, bstep = TB ? 128u : 2u;
    const uint32_t a_wg = wg * (TA ? SLAB_BYTES : 64u * 128u);
    float d[BN / 2];
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      uint32_t prev_stage = 0;
      // zero the accumulator here rather than through wgmma's scale-d: its registers are then dead between the
      // shared-memory store of one tile and the start of the next
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      for (int kb = t.kb0; kb < t.kb1; ++kb) {
        mbar_wait_mma(full_bar + 8 * stage, phase);
        const uint32_t a_base = sA + stage * A_BYTES + a_wg;
        const uint32_t b_base = sB + stage * G_B_BYTES;
        const uint64_t ad0 = smem_desc_sw128(a_base, TA ? SLAB_BYTES : 0u, 1024);
        const uint64_t bd0 = smem_desc_sw128(b_base, TB ? SLAB_BYTES : 0u, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          wgmma_m64n128<TA, TB>(d, ad0 + k * astep, bd0 + k * bstep, 1u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage goes back to the producer
        if (kb > t.kb0 && (threadIdx.x & 127) == 0) mbar_arrive(empty_bar + 8 * prev_stage);
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(empty_bar + 8 * prev_stage);
      // the epilogue has finished reading the previous tile (it signals EMPTY after every tile but the last)
      if (tile != blockIdx.x) named_bar_sync(G_BAR_EMPTY, G_BAR_HANDOFF_THREADS);
      acc_store_smem<BN>(d, sAcc >> 2, 64 * wg);
      named_bar_arrive(G_BAR_FULL, G_BAR_HANDOFF_THREADS);
    }
  } else {
    // ------------------------------------------------------------------ epilogue warpgroup
    setmaxnreg_inc<G_REGS_EPI>();
    const int ew = warp - 12;      // rows [32 ew, 32 ew + 32) of the tile, one per lane
    constexpr int CH = BN / 64;    // 32-column chunks per half tile
    const uint32_t stg = stg_base + ew * STG_BYTES;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int row0 = t.m_blk * BM + ew * 32;
      const int row = row0 + lane;
      const bool row_ok = row < p.M;
      const int n0 = t.n_blk * BN;
      // pull this tile's bias into L1 and the per-element operands (ReLU mask / residual rows) into L2 while the
      // accumulator is being produced
      if (p.bias && lane < BN / 32 && n0 + lane * 32 < p.N)
        asm volatile("prefetch.global.L1 [%0];" ::"l"(p.bias + n0 + lane * 32));
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int cbase = n0 + half * (BN / 2);
        if (row_ok && cbase < p.N) {
          if (p.aux) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.aux + (long long)row * p.ldaux + cbase));
          if (p.residual) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.residual + (long long)row * p.ldr + cbase));
        }
      }
      named_bar_sync(G_BAR_FULL, G_BAR_HANDOFF_THREADS);
#pragma unroll 1
      for (int half = 0; half < 2; ++half) {  // columns [half * BN/2, (half + 1) * BN/2) of the tile
        const int cbase = n0 + half * (BN / 2);
        const uint32_t t_addr = (sAcc >> 2) + (ew * 32 + lane) * BN + half * (BN / 2);
        if constexpr (WCE) {
          epi_ce_grad_weighted<CH>(p, t_addr, row, row_ok, cbase, stg, row0, lane);
          continue;
        }
        if constexpr (MLP == G_GELU_FWD) {
          epi_gelu_store<CH>(p, t_addr, cbase, stg, row0, lane);
          continue;
        }
        if constexpr (MLP == G_GELU_BWD) {
          epi_gelu_bwd<CH>(p, t_addr, cbase, stg, row0, lane);
          continue;
        }
        if constexpr (glu_fwd(MLP)) {  // the whole tile at once: value and gate halves of the same 64 columns
          if (half == 0) epi_glu_store<MLP == G_GLU_GELU_FWD>(p, t_addr, t.n_blk * 64, stg, row0, lane);
          continue;
        }
        if constexpr (glu_bwd(MLP)) {
          epi_glu_bwd<MLP == G_GLU_GELU_BWD>(p, t_addr, cbase, stg, row0, lane);
          continue;
        }
        switch (p.mode) {
          case DB200_EPI_STORE:    epi_store<CH, DROP>(p, t_addr, row, row_ok, cbase, stg, row0, lane); break;
          case DB200_EPI_ATOMIC:
            epi_atomic<CH>(p, reinterpret_cast<float*>(p.D) + (long long)t.split * p.M * p.ldd, row, row_ok, cbase,
                           t_addr);
            break;
          case DB200_EPI_RELU_BWD: epi_relu_bwd<CH>(p, t_addr, row, row_ok, cbase, stg, row0, lane); break;
          case DB200_EPI_CE_STATS: epi_ce_stats<CH>(p, t_addr, row, row_ok, cbase, t.n_blk * 2 + half); break;
          case DB200_EPI_CE_GRAD:  epi_ce_grad<CH>(p, t_addr, row, row_ok, cbase, stg, row0, lane); break;
          default: break;
        }
      }
      if (tile + (int)gridDim.x < total_tiles) named_bar_arrive(G_BAR_EMPTY, G_BAR_HANDOFF_THREADS);
    }
  }
}

// ----------------------------------------------------------------------------------------------------------------------
// The ping-pong kernel for short contractions (gemm_run picks it by K and epilogue).  With K <= 1024 a tile's mainloop
// is at most 16 k-blocks, and the hand-off above (128 x 128 fp32 through shared memory, both MMA warpgroups storing at
// once, one epilogue warp per SM sub-partition) costs about as much as the mainloop.  Here each of the two consumer
// warpgroups owns a whole 128 x 128 tile: two m64n128 chains per k-step against the same B descriptor, 128 accumulators
// per thread.  The CTA's tiles alternate between the warpgroups, a pair of named barriers gives the tensor cores to one
// warpgroup at a time, and a warpgroup runs its epilogue from its registers (gemm_common.cuh: fragment epilogues) while
// the other multiplies.  The shared memory the accumulator tile took goes to the operand ring.
//
//   warp 0     : TMA producer, filling stages in consumption order (the tiles of warpgroup 0 and 1 interleaved)
//   warps 1-3  : idle (they hand their registers to the consumers and exit)
//   warps 4-7  : consumer warpgroup 0: entries 0, 2, 4, ... of the CTA's tile list
//   warps 8-11 : consumer warpgroup 1: entries 1, 3, 5, ...
// ----------------------------------------------------------------------------------------------------------------------
constexpr int PP_THREADS = 384;
constexpr int PP_STAGES = 6;
constexpr size_t PP_SMEM_BYTES =
    1024 /*align slack*/ + size_t(PP_STAGES) * G_STAGE_BYTES + 256 /*barriers*/ + 8 * STG_BYTES;
static_assert(PP_SMEM_BYTES <= 227 * 1024, "ping-pong GEMM shared memory exceeds the H100 per-block limit");
// 384 threads compile to 168 registers each; the producer warpgroup's share goes to the consumers (128 accumulators)
constexpr int PP_REGS_PRODUCER = 40, PP_REGS_MMA = 232;
static_assert(128 * PP_REGS_PRODUCER + 256 * PP_REGS_MMA <= 384 * 168, "ping-pong GEMM register budget");
// named barriers: PP_BAR_TURN + g admits warpgroup g to the tensor cores (its 128 threads wait, the other warpgroup's
// 128 arrive); PP_BAR_PAIR + 2 g + {0, 1}: the two warp pairs of warpgroup g around their staging blocks
constexpr int PP_BAR_TURN = 1, PP_BAR_PAIR = 3;

// The epilogues of gemm_pp_kernel: STORE without dropout, RELU_BWD and plain CE_GRAD, whose per-element results do not
// depend on which thread holds an element.  CE_STATS sums a row's exponentials in column order, which a thread of the
// accumulator fragment cannot do (it holds two columns in eight), so it stays with the row-per-thread epilogue: lse,
// and with it every gradient behind it, keeps its bits.
static bool pp_has_epilogue(int mode, bool drop, bool wce, int gelu) {
  return !drop && !wce && !gelu && (mode == DB200_EPI_STORE || mode == DB200_EPI_RELU_BWD || mode == DB200_EPI_CE_GRAD);
}
// Up to this many k-blocks per tile a product runs on gemm_pp_kernel (K <= 1024).  -DDB200_PP_MAX_KB=<n> moves the
// rule in a side build, for measuring both kernels at one K (tools/bench_gemm_shapes.py).
#ifndef DB200_PP_MAX_KB
#define DB200_PP_MAX_KB 16
#endif
constexpr int PP_MAX_KB = DB200_PP_MAX_KB;

template <int TA, int TB>
__global__ void __launch_bounds__(PP_THREADS, 1)
gemm_pp_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  constexpr int BN = GBN;
  constexpr int STAGES = PP_STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t sA = (raw + 1023u) & ~1023u;  // SWIZZLE_128B tiles need 1024-byte alignment
  const uint32_t sB = sA + STAGES * A_BYTES;
  const uint32_t bars = sA + STAGES * G_STAGE_BYTES;
  const uint32_t full_bar = bars;                // STAGES x 8 B
  const uint32_t empty_bar = bars + 8 * STAGES;  // STAGES x 8 B
  const uint32_t stg_base = bars + 256;          // 2 warpgroups x 4 x STG_BYTES, 256-byte aligned

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(full_bar + 8 * i, 1);
      mbar_init(empty_bar + 8 * i, 1);  // a stage is read by one warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int total_tiles = p.m_tiles * p.n_tiles;  // never split-K: every tile has p.kb_total k-blocks

  if (warp < 4) {
    setmaxnreg_dec<PP_REGS_PRODUCER>();
    if (warp != 0) return;
    // ------------------------------------------------------------------ TMA producer (as in gemm_tc_kernel)
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int m0 = t.m_blk * BM, n0 = t.n_blk * BN;
      for (int kb = 0; kb < p.kb_total; ++kb) {
        mbar_wait_mma(empty_bar + 8 * stage, phase ^ 1);
        const uint32_t fb = full_bar + 8 * stage;
        if (elect_one_sync()) {
          mbar_expect_tx(fb, G_STAGE_BYTES);
          const int k0 = kb * BK;
          const uint32_t a_dst = sA + stage * A_BYTES;
          const uint32_t b_dst = sB + stage * G_B_BYTES;
          if (p.a_3d) {
            tma_load_3d(a_dst, &tmA, fb, 0, k0, m0 >> 6);
          } else if (p.a_mn) {
#pragma unroll
            for (int s = 0; s < BM / 64; ++s) tma_load_2d(a_dst + s * SLAB_BYTES, &tmA, fb, m0 + 64 * s, k0);
          } else {
            tma_load_2d(a_dst, &tmA, fb, k0, m0);
          }
          if (p.b_3d) {
            tma_load_3d(b_dst, &tmB, fb, 0, k0, n0 >> 6);
          } else if (p.b_mn) {
#pragma unroll
            for (int s = 0; s < BN / 64; ++s) tma_load_2d(b_dst + s * SLAB_BYTES, &tmB, fb, n0 + 64 * s, k0);
          } else {
            tma_load_2d(b_dst, &tmB, fb, k0, n0);
          }
        }
        __syncwarp();
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumer warpgroups
    setmaxnreg_inc<PP_REGS_MMA>();
    const int wg = (warp - 4) >> 2;
    const FragCtx f = frag_ctx<0>(stg_base + wg * 4 * STG_BYTES, threadIdx.x & 127, PP_BAR_PAIR + 2 * wg);
    constexpr uint64_t astep = TA ? 128u : 2u, bstep = TB ? 128u : 2u;
    constexpr uint32_t a_chain = TA ? SLAB_BYTES : 64u * 128u;  // rows 64-127 of the A stage
    float d[2 * (BN / 2)];
    for (int j = wg; blockIdx.x + (long long)j * gridDim.x < total_tiles; j += 2) {
      const int tile = blockIdx.x + j * gridDim.x;
      const TileCoord t = decode_tile(p, tile);
      // ring position of this tile's first k-block: the other warpgroup consumed the tiles in between
      const uint32_t it = (uint32_t)j * (uint32_t)p.kb_total;
      uint32_t stage = it % STAGES, phase = (it / STAGES) & 1u, prev_stage = 0;
#pragma unroll
      for (int i = 0; i < 2 * (BN / 2); ++i) d[i] = 0.f;
      // the other warpgroup has issued the last MMA of the tile before this one
      if (j > 0) named_bar_sync(PP_BAR_TURN + wg, 256);
      for (int kb = 0; kb < p.kb_total; ++kb) {
        mbar_wait_mma(full_bar + 8 * stage, phase);
        const uint64_t ad0 = smem_desc_sw128(sA + stage * A_BYTES, TA ? SLAB_BYTES : 0u, 1024);
        const uint64_t ad1 = smem_desc_sw128(sA + stage * A_BYTES + a_chain, TA ? SLAB_BYTES : 0u, 1024);
        const uint64_t bd0 = smem_desc_sw128(sB + stage * G_B_BYTES, TB ? SLAB_BYTES : 0u, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          wgmma_m64n128<TA, TB>(d, ad0 + k * astep, bd0 + k * bstep, 1u);
          wgmma_m64n128<TA, TB>(d + BN / 2, ad1 + k * astep, bd0 + k * bstep, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage goes back to the producer
        if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(empty_bar + 8 * prev_stage);
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      // one arrival per wait: only when the other warpgroup has a tile after this one
      if (tile + (int)gridDim.x < total_tiles) named_bar_arrive(PP_BAR_TURN + (wg ^ 1), 256);
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(empty_bar + 8 * prev_stage);
      const int m0 = t.m_blk * BM, n0 = t.n_blk * BN;
      switch (p.mode) {
        case DB200_EPI_STORE:    frag_store<0>(p, d, f, m0, n0); break;
        case DB200_EPI_RELU_BWD: frag_relu_bwd<0>(p, d, f, m0, n0); break;
        case DB200_EPI_CE_GRAD:  frag_ce_grad(p, d, f, m0, n0); break;
        default: break;
      }
    }
  }
}

template <int TA, int TB>
static int launch_gemm_pp(cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p) {
  static const cudaError_t attr_rc = cudaFuncSetAttribute(gemm_pp_kernel<TA, TB>,
                                                          cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                          (int)PP_SMEM_BYTES);  // once, thread-safe (magic static)
  DB200_CUDA(attr_rc);
  const int total = p.m_tiles * p.n_tiles;
  const int grid = total < sm_count() ? total : sm_count();
  gemm_pp_kernel<TA, TB><<<grid, PP_THREADS, PP_SMEM_BYTES, stream>>>(tmA, tmB, p);
  return check_launch("gemm_pp_kernel");
}

// ----------------------------------------------------------------------------------------------------------------------
// The wide kernel for long contractions (gemm_run picks it by K, epilogue and tile count).  A 128 x 128 tile loads
// (128 + 128) x K bf16 operands from L2 for 2 x 128 x 128 x K FLOP; a 128 x 256 tile loads (128 + 256) x K for twice
// the FLOP, a quarter less L2 -> shared-memory traffic per FLOP, and the long-K products on 128 x 128 tiles level off
// near 10 TB/s of it (DESIGN.md §3).  Warpgroup g issues wgmma m64n256 for rows [64 g, 64 g + 64) of the tile (128
// accumulators per thread) and, when the tile's mainloop is done, runs its epilogue from those registers
// (gemm_common.cuh: fragment epilogues, chains side by side).  The epilogue overlaps only the producer's loads for
// the next tile, not its MMAs.  Each element gets the k16 steps of gemm_tc_kernel in the same k-block order and the
// same per-element epilogue expression.
//
//   warp 0     : TMA producer              smem ring: W_STAGES x {A 128x64, B 256x64} bf16 (48 KiB per stage)
//   warps 1-3  : idle (they hand their registers to the consumers and exit)
//   warps 4-11 : two MMA warpgroups, rows [64 g, 64 g + 64) of every tile of the CTA
// ----------------------------------------------------------------------------------------------------------------------
constexpr int WBN = 256;
constexpr int W_STAGES = 4;
constexpr uint32_t W_B_BYTES = WBN * BK * 2;
constexpr uint32_t W_STAGE_BYTES = A_BYTES + W_B_BYTES;
constexpr size_t W_SMEM_BYTES =
    1024 /*align slack*/ + size_t(W_STAGES) * W_STAGE_BYTES + 256 /*barriers*/ + 8 * STG_BYTES;
static_assert(W_SMEM_BYTES <= 227 * 1024, "wide GEMM shared memory exceeds the H100 per-block limit");
// named barriers: W_BAR_PAIR + 2 g + {0, 1}: the two warp pairs of warpgroup g around their staging blocks
constexpr int W_BAR_PAIR = 1;

// STORE without dropout and RELU_BWD.  The single-split ATOMIC vocabulary wgrad (both operands MN-major) measured
// no faster on 128 x 256 tiles, and split-K, CE, GELU and dropout products stay with their kernels.
static bool wide_has_epilogue(int mode, bool drop, bool wce, int gelu) {
  return !drop && !wce && !gelu && (mode == DB200_EPI_STORE || mode == DB200_EPI_RELU_BWD);
}
// A product needs at least this many 128 x 256 tiles per SM for the wide kernel: at one tile per SM it measured as
// fast as the 128 x 128 kernel, from two on 1.15x and more.  -DDB200_WIDE_MIN_TILES=<n> moves the rule in a side
// build (tools/bench_gemm_shapes.py --sweep).
#ifndef DB200_WIDE_MIN_TILES
#define DB200_WIDE_MIN_TILES 2
#endif
constexpr int WIDE_MIN_TILES = DB200_WIDE_MIN_TILES;

template <int TA, int TB>
__global__ void __launch_bounds__(PP_THREADS, 1)
gemm_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  constexpr int STAGES = W_STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t sA = (raw + 1023u) & ~1023u;  // SWIZZLE_128B tiles need 1024-byte alignment
  const uint32_t sB = sA + STAGES * A_BYTES;
  const uint32_t bars = sA + STAGES * W_STAGE_BYTES;
  const uint32_t full_bar = bars;                // STAGES x 8 B
  const uint32_t empty_bar = bars + 8 * STAGES;  // STAGES x 8 B
  const uint32_t stg_base = bars + 256;          // 2 warpgroups x 4 x STG_BYTES, 256-byte aligned

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(full_bar + 8 * i, 1);
      mbar_init(empty_bar + 8 * i, 2);  // one arrive per MMA warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int total_tiles = p.m_tiles * p.n_tiles;  // n_tiles counts 256-wide tiles; never split-K

  if (warp < 4) {
    setmaxnreg_dec<PP_REGS_PRODUCER>();
    if (warp != 0) return;
    // ------------------------------------------------------------------ TMA producer
    // the tensor maps are gemm_tc_kernel's (B boxes of 128 rows or 2 slabs): a 256-wide B stage takes two of them
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int m0 = t.m_blk * BM, n0 = t.n_blk * WBN;
      for (int kb = 0; kb < p.kb_total; ++kb) {
        mbar_wait_mma(empty_bar + 8 * stage, phase ^ 1);
        const uint32_t fb = full_bar + 8 * stage;
        if (elect_one_sync()) {
          mbar_expect_tx(fb, W_STAGE_BYTES);
          const int k0 = kb * BK;
          const uint32_t a_dst = sA + stage * A_BYTES;
          const uint32_t b_dst = sB + stage * W_B_BYTES;
          if (p.a_3d) {
            tma_load_3d(a_dst, &tmA, fb, 0, k0, m0 >> 6);
          } else if (p.a_mn) {
#pragma unroll
            for (int s = 0; s < BM / 64; ++s) tma_load_2d(a_dst + s * SLAB_BYTES, &tmA, fb, m0 + 64 * s, k0);
          } else {
            tma_load_2d(a_dst, &tmA, fb, k0, m0);
          }
          if (p.b_3d) {
#pragma unroll
            for (int s = 0; s < WBN / GBN; ++s)
              tma_load_3d(b_dst + s * G_B_BYTES, &tmB, fb, 0, k0, (n0 >> 6) + s * (GBN / 64));
          } else if (p.b_mn) {
#pragma unroll
            for (int s = 0; s < WBN / 64; ++s) tma_load_2d(b_dst + s * SLAB_BYTES, &tmB, fb, n0 + 64 * s, k0);
          } else {
#pragma unroll
            for (int s = 0; s < WBN / GBN; ++s) tma_load_2d(b_dst + s * G_B_BYTES, &tmB, fb, k0, n0 + GBN * s);
          }
        }
        __syncwarp();
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ------------------------------------------------------------------ MMA warpgroups
    setmaxnreg_inc<PP_REGS_MMA>();
    const int wg = (warp - 4) >> 2;  // rows [64 wg, 64 wg + 64) of every tile
    const FragCtx f = frag_ctx<WBN / 2>(stg_base + wg * 4 * STG_BYTES, threadIdx.x & 127, W_BAR_PAIR + 2 * wg);
    constexpr uint64_t astep = TA ? 128u : 2u, bstep = TB ? 128u : 2u;
    const uint32_t a_wg = wg * (TA ? SLAB_BYTES : 64u * 128u);
    float d[WBN / 2];
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      uint32_t prev_stage = 0;
#pragma unroll
      for (int i = 0; i < WBN / 2; ++i) d[i] = 0.f;
      for (int kb = 0; kb < p.kb_total; ++kb) {
        mbar_wait_mma(full_bar + 8 * stage, phase);
        const uint64_t ad0 = smem_desc_sw128(sA + stage * A_BYTES + a_wg, TA ? SLAB_BYTES : 0u, 1024);
        const uint64_t bd0 = smem_desc_sw128(sB + stage * W_B_BYTES, TB ? SLAB_BYTES : 0u, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          wgmma_m64n256<TA, TB>(d, ad0 + k * astep, bd0 + k * bstep, 1u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage goes back to the producer
        if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(empty_bar + 8 * prev_stage);
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(empty_bar + 8 * prev_stage);
      const int m0 = t.m_blk * BM + 64 * wg, n0 = t.n_blk * WBN;
      switch (p.mode) {
        case DB200_EPI_STORE:    frag_store<WBN / 2>(p, d, f, m0, n0); break;
        case DB200_EPI_RELU_BWD: frag_relu_bwd<WBN / 2>(p, d, f, m0, n0); break;
        default: break;
      }
    }
  }
}

template <int TA, int TB>
static int launch_gemm_wide(cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB, GemmParams p) {
  static const cudaError_t attr_rc = cudaFuncSetAttribute(gemm_wide_kernel<TA, TB>,
                                                          cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                          (int)W_SMEM_BYTES);  // once, thread-safe (magic static)
  DB200_CUDA(attr_rc);
  p.n_tiles = (p.N + WBN - 1) / WBN;
  const int total = p.m_tiles * p.n_tiles;
  const int grid = total < sm_count() ? total : sm_count();
  gemm_wide_kernel<TA, TB><<<grid, PP_THREADS, W_SMEM_BYTES, stream>>>(tmA, tmB, p);
  return check_launch("gemm_wide_kernel");
}

template <int TA, int TB, bool DROP, bool WCE = false, int MLP = 0>
static int launch_gemm(cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p) {
  static const cudaError_t attr_rc = cudaFuncSetAttribute(gemm_tc_kernel<TA, TB, DROP, WCE, MLP>,
                                                          cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                          (int)G_SMEM_BYTES);  // once, thread-safe (magic static)
  DB200_CUDA(attr_rc);
  const int total = p.m_tiles * p.n_tiles * p.splits;
  const int grid = total < sm_count() ? total : sm_count();
  gemm_tc_kernel<TA, TB, DROP, WCE, MLP><<<grid, GEMM_THREADS, G_SMEM_BYTES, stream>>>(tmA, tmB, p);
  return check_launch("gemm_tc_kernel");
}

}  // namespace db200

using namespace db200;

extern "C" int db200_gemm_ce_tiles(int N) { return 2 * ((N + GBN - 1) / GBN); }

// K splits of an ATOMIC product (1 for every other mode)
static int gemm_splits(int M, int N, int K, const db200_gemm_epilogue* epi) {
  if (epi->mode != DB200_EPI_ATOMIC) return 1;
  const int kb_total = (K + BK - 1) / BK;
  int splits = epi->split_k;
  if (splits <= 0) {  // auto: fill the machine, keep >= 4 k-blocks per split
    const int tiles = ((M + BM - 1) / BM) * ((N + GBN - 1) / GBN);
    splits = sm_count() / (tiles > 0 ? tiles : 1);
    if (splits > kb_total / 4) splits = kb_total / 4;
    if (splits < 1) splits = 1;
  }
  if (splits > kb_total) splits = kb_total;
  if (splits < 1) splits = 1;
  // every split must own at least one k-block
  const int per = (kb_total + splits - 1) / splits;
  return (kb_total + per - 1) / per;
}

extern "C" int64_t db200_gemm_workspace_bytes(int M, int N, int K, const db200_gemm_epilogue* epi) {
  if (!epi || M <= 0 || N <= 0 || K <= 0) return 0;
  const int splits = gemm_splits(M, N, K, epi);
  if (splits > 1) return (int64_t)splits * M * N * (int64_t)sizeof(float);
  const bool colsum = (epi->mode == DB200_EPI_CE_GRAD || epi->mode == DB200_EPI_RELU_BWD) && epi->colsum;
  if (colsum) return (int64_t)((M + BM - 1) / BM) * (BM / 32) * N * (int64_t)sizeof(float);
  return 0;
}

extern "C" int db200_gemm_bf16(db200_stream_t stream_, const void* A, int a_mn_major, int64_t lda, const void* B,
                               int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M, int N, int K,
                               const db200_gemm_epilogue* epi) {
  return db200_gemm_bf16_ex(stream_, A, a_mn_major, lda, B, b_mn_major, ldb, D, ldd, M, N, K, epi, nullptr);
}

// every product: cew != NULL selects the weighted CE_GRAD epilogue (validated by db200_gemm_bf16_ce_weighted), gelu the
// GELU MLP's store (G_GELU_FWD, pre-activation output z / ldz) or dgrad (G_GELU_BWD) epilogue (validated by
// db200_gemm_bf16_gelu / db200_gemm_bf16_gelu_bwd), or the gated MLP's (G_GLU_*, validated by db200_gemm_bf16_glu /
// db200_gemm_bf16_glu_bwd; N is the h width, B of the forward and D / aux / colsum of the backward are 2N wide)
static int gemm_run(db200_stream_t stream_, const void* A, int a_mn_major, int64_t lda, const void* B, int b_mn_major,
                    int64_t ldb, void* D, int64_t ldd, int M, int N, int K, const db200_gemm_epilogue* epi,
                    const db200_dropout* dropout, const db200_ce_weights* cew, int gelu = 0, void* z = nullptr,
                    int64_t ldz = 0) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(epi != nullptr, DB200_E_INVALID, "gemm: epilogue descriptor is NULL");
  const bool drop = dropout_active(dropout);
  DB200_REQUIRE(!drop || epi->mode == DB200_EPI_STORE, DB200_E_INVALID, "gemm: dropout needs the STORE epilogue");
  DB200_REQUIRE(M > 0 && N > 0 && K > 0, DB200_E_INVALID, "gemm: M,N,K must be positive (got %d,%d,%d)", M, N, K);
  DB200_REQUIRE(A && B, DB200_E_INVALID, "gemm: NULL operand");
  DB200_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, DB200_E_ALIGN,
                "gemm: lda/ldb must be multiples of 8 elements (16 B) for TMA (got %lld, %lld)", (long long)lda,
                (long long)ldb);
  DB200_REQUIRE(lda >= (a_mn_major ? M : K) && ldb >= (b_mn_major ? N : K), DB200_E_INVALID,
                "gemm: leading dimension smaller than the contiguous extent");
  const int mode = epi->mode;
  DB200_REQUIRE(mode >= DB200_EPI_STORE && mode <= DB200_EPI_CE_GRAD, DB200_E_INVALID, "gemm: unknown epilogue %d",
                mode);
  if (mode != DB200_EPI_CE_STATS) {
    DB200_REQUIRE(D != nullptr && aligned16(D), DB200_E_ALIGN, "gemm: D must be non-NULL and 16-byte aligned");
    DB200_REQUIRE(ldd >= N, DB200_E_INVALID, "gemm: ldd < N");
  }
  if (mode == DB200_EPI_STORE || mode == DB200_EPI_RELU_BWD || mode == DB200_EPI_CE_GRAD) {
    DB200_REQUIRE(N % 8 == 0 && ldd % 8 == 0, DB200_E_ALIGN,
                  "gemm: vectorised store epilogues need N and ldd to be multiples of 8 (got N=%d ldd=%lld)", N,
                  (long long)ldd);
  }
  DB200_REQUIRE(aligned16(epi->bias), DB200_E_ALIGN, "gemm: bias must be 16-byte aligned");
  if (mode == DB200_EPI_STORE && epi->residual)
    DB200_REQUIRE(aligned16(epi->residual) && epi->ldr % 8 == 0 && epi->ldr >= N, DB200_E_ALIGN,
                  "gemm: residual must be 16-byte aligned with ldr %% 8 == 0");
  if (mode == DB200_EPI_RELU_BWD)
    DB200_REQUIRE(epi->aux && aligned16(epi->aux) && epi->ldaux % 8 == 0 && epi->ldaux >= N, DB200_E_ALIGN,
                  "gemm: RELU_BWD needs an aligned aux tensor");
  if (mode == DB200_EPI_CE_STATS)
    DB200_REQUIRE(epi->labels && epi->part_max && epi->part_sum && epi->label_logit && epi->n_valid > 0 &&
                      epi->n_valid <= N,
                  DB200_E_INVALID, "gemm: CE_STATS needs labels/part_max/part_sum/label_logit and 0 < n_valid <= N");
  if (mode == DB200_EPI_CE_GRAD)
    DB200_REQUIRE(epi->labels && epi->lse && epi->n_valid > 0 && epi->n_valid <= N && (cew || epi->alpha > 0.f),
                  DB200_E_INVALID, "gemm: CE_GRAD needs labels/lse, 0 < n_valid <= N and alpha > 0");
  DB200_REQUIRE(mode == DB200_EPI_ATOMIC || epi->split_k <= 1, DB200_E_INVALID,
                "gemm: split_k > 1 is only valid with DB200_EPI_ATOMIC");
  const int splits = gemm_splits(M, N, K, epi);
  const int kb_total = (K + BK - 1) / BK;
  const int n_sums = glu_bwd(gelu) ? 2 * N : N;  // columns of the fused column sums
  DB200_REQUIRE(workspace_ok(epi->workspace, epi->workspace_bytes, db200_gemm_workspace_bytes(M, n_sums, K, epi)),
                DB200_E_INVALID, "gemm: needs an aligned epi->workspace of db200_gemm_workspace_bytes() bytes");

  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.a_mn = a_mn_major ? 1 : 0;
  p.b_mn = b_mn_major ? 1 : 0;
  p.m_tiles = (M + BM - 1) / BM;
  p.splits = splits;
  p.kb_total = kb_total;
  p.mode = mode;
  p.out_f32 = epi->out_f32;
  p.relu = epi->relu;
  p.alpha = epi->alpha;
  p.D = D;
  p.ldd = ldd;
  p.bias = epi->bias;
  p.residual = reinterpret_cast<const bf16*>(epi->residual);
  p.ldr = epi->ldr;
  p.aux = reinterpret_cast<const bf16*>(epi->aux);
  p.ldaux = epi->ldaux;
  p.labels = epi->labels;
  p.part_max = epi->part_max;
  p.part_sum = epi->part_sum;
  p.label_logit = epi->label_logit;
  p.lse = epi->lse;
  p.n_valid = epi->n_valid;
  p.colsum = (mode == DB200_EPI_CE_GRAD || mode == DB200_EPI_RELU_BWD) ? epi->colsum : nullptr;
  p.drop = drop ? *dropout : db200_dropout{};
  p.cew = cew ? *cew : db200_ce_weights{};
  p.zout = reinterpret_cast<bf16*>(z);
  p.ldz = ldz;

  p.n_tiles = glu_fwd(gelu) ? N / 64 : (N + GBN - 1) / GBN;
  p.n_parts = 2 * p.n_tiles;

  // MN-major operands whose MN extent is a multiple of 64: one rank-3 map {64, K, MN/64} (stride of the slab index =
  // 128 bytes) fetches every 64-wide slab of a stage with a single TMA instruction instead of one per slab.
  p.a_3d = (p.a_mn && M % 64 == 0) ? 1 : 0;
  p.b_3d = (p.b_mn && N % 64 == 0 && !glu_fwd(gelu)) ? 1 : 0;
  CUtensorMap tmA, tmB;
  int rc;
  if (p.a_3d) {
    uint64_t dims[3] = {64, (uint64_t)K, (uint64_t)M / 64};
    uint64_t str[2] = {(uint64_t)lda * 2, 128};
    uint32_t box[3] = {64, BK, 2};
    rc = make_tmap_bf16(&tmA, A, 3, dims, str, box);
  } else if (p.a_mn) rc = make_tmap_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 64, BK);
  else               rc = make_tmap_2d(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, BM);
  if (rc != DB200_OK) return rc;
  if (p.b_3d) {
    uint64_t dims[3] = {64, (uint64_t)K, (uint64_t)N / 64};
    uint64_t str[2] = {(uint64_t)ldb * 2, 128};
    uint32_t box[3] = {64, BK, GBN / 64};
    rc = make_tmap_bf16(&tmB, B, 3, dims, str, box);
  } else if (p.b_mn) {  // a GLU forward's B holds 2N columns: value slabs, then gate slabs
    rc = make_tmap_2d(&tmB, B, (uint64_t)(glu_fwd(gelu) ? 2 * N : N), (uint64_t)K, (uint64_t)ldb, 64, BK);
  }
  else               rc = make_tmap_2d(&tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, BK, GBN);
  if (rc != DB200_OK) return rc;

  // Sums over tiles go through a workspace and are added in a fixed order after the GEMM (run-to-run identical results):
  // the per-split slices of a split-K product, and the per-32-row-block column sums of the fused bias gradient.
  float* const colsum_out = p.colsum;
  float* const d_out = reinterpret_cast<float*>(D);
  const int row_blocks = p.m_tiles * (BM / 32);
  if (p.splits > 1) {
    p.D = epi->workspace;
    p.ldd = N;
  } else if (colsum_out) {
    p.colsum = static_cast<float*>(epi->workspace);
  }
  // Short contractions with a fragment epilogue run on the ping-pong kernel.  The rule reads the epilogue, K and the
  // operand majors only, never M: prefill (M = B P) and training (M = B S) must take the same path, bit for bit.
  // Long ones with enough tiles run on the wide kernel, which gives every element gemm_tc_kernel's bits.
  const int wide_tiles = p.m_tiles * ((N + WBN - 1) / WBN);
  if (kb_total <= PP_MAX_KB && pp_has_epilogue(mode, drop, cew != nullptr, gelu)) {
    if (p.a_mn) rc = p.b_mn ? launch_gemm_pp<1, 1>(stream, tmA, tmB, p) : launch_gemm_pp<1, 0>(stream, tmA, tmB, p);
    else        rc = p.b_mn ? launch_gemm_pp<0, 1>(stream, tmA, tmB, p) : launch_gemm_pp<0, 0>(stream, tmA, tmB, p);
  } else if (kb_total > PP_MAX_KB && wide_has_epilogue(mode, drop, cew != nullptr, gelu) &&
             wide_tiles >= WIDE_MIN_TILES * sm_count()) {
    if (p.a_mn) rc = p.b_mn ? launch_gemm_wide<1, 1>(stream, tmA, tmB, p) : launch_gemm_wide<1, 0>(stream, tmA, tmB, p);
    else        rc = p.b_mn ? launch_gemm_wide<0, 1>(stream, tmA, tmB, p) : launch_gemm_wide<0, 0>(stream, tmA, tmB, p);
  } else if (gelu == G_GELU_FWD)   // the MLP's W1 forward: A k-major, B mn-major
    rc = (!p.a_mn && p.b_mn) ? launch_gemm<0, 1, false, false, G_GELU_FWD>(stream, tmA, tmB, p)
                             : set_error(DB200_E_UNSUPPORTED, "gemm_gelu: needs a k-major A and an mn-major B");
  else if (gelu == G_GELU_BWD)   // its dgrad dH = dbranch W2^T: both k-major
    rc = (!p.a_mn && !p.b_mn) ? launch_gemm<0, 0, false, false, G_GELU_BWD>(stream, tmA, tmB, p)
                              : set_error(DB200_E_UNSUPPORTED, "gemm_gelu_bwd: needs k-major A and B");
  else if (glu_fwd(gelu))   // the gated MLP's W1 forward: A k-major, B mn-major
    rc = (p.a_mn || !p.b_mn) ? set_error(DB200_E_UNSUPPORTED, "gemm_glu: needs a k-major A and an mn-major B")
         : gelu == G_GLU_GELU_FWD ? launch_gemm<0, 1, false, false, G_GLU_GELU_FWD>(stream, tmA, tmB, p)
                                  : launch_gemm<0, 1, false, false, G_GLU_RELU_FWD>(stream, tmA, tmB, p);
  else if (glu_bwd(gelu))   // its dgrad dh = dbranch W2^T: both k-major
    rc = (p.a_mn || p.b_mn) ? set_error(DB200_E_UNSUPPORTED, "gemm_glu_bwd: needs k-major A and B")
         : gelu == G_GLU_GELU_BWD ? launch_gemm<0, 0, false, false, G_GLU_GELU_BWD>(stream, tmA, tmB, p)
                                  : launch_gemm<0, 0, false, false, G_GLU_RELU_BWD>(stream, tmA, tmB, p);
  else if (cew)     // the vocabulary product: A k-major, B mn-major (wout) or k-major (a tied wte)
    rc = p.a_mn ? set_error(DB200_E_UNSUPPORTED, "gemm: weighted CE_GRAD needs a k-major A (and a B of either major)")
         : p.b_mn ? launch_gemm<0, 1, false, true>(stream, tmA, tmB, p) : launch_gemm<0, 0, false, true>(stream, tmA, tmB, p);
  else if (drop)    // residual dropout runs in forward products only: A k-major, B mn-major
    rc = (!p.a_mn && p.b_mn) ? launch_gemm<0, 1, true>(stream, tmA, tmB, p)
                             : set_error(DB200_E_UNSUPPORTED, "gemm: dropout needs a k-major A and an mn-major B");
  else if (p.a_mn) rc = p.b_mn ? launch_gemm<1, 1, false>(stream, tmA, tmB, p) : launch_gemm<1, 0, false>(stream, tmA, tmB, p);
  else             rc = p.b_mn ? launch_gemm<0, 1, false>(stream, tmA, tmB, p) : launch_gemm<0, 0, false>(stream, tmA, tmB, p);
  if (rc != DB200_OK) return rc;
  if (p.splits > 1) return reduce_splits_add(stream, static_cast<const float*>(p.D), p.splits, M, N, d_out, ldd);
  if (colsum_out) return reduce_rows_add(stream, p.colsum, row_blocks, n_sums, colsum_out);
  return DB200_OK;
}

extern "C" int db200_gemm_bf16_ex(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda, const void* B,
                                  int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M, int N, int K,
                                  const db200_gemm_epilogue* epi, const db200_dropout* dropout) {
  return gemm_run(stream, A, a_mn_major, lda, B, b_mn_major, ldb, D, ldd, M, N, K, epi, dropout, nullptr);
}

extern "C" int db200_gemm_bf16_ce_weighted(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda,
                                           const void* B, int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M,
                                           int N, int K, const db200_gemm_epilogue* epi, const db200_ce_weights* w) {
  DB200_REQUIRE(epi != nullptr && epi->mode == DB200_EPI_CE_GRAD, DB200_E_INVALID,
                "gemm_ce_weighted: needs an epilogue descriptor with mode DB200_EPI_CE_GRAD");
  const int rc = ce_weights_check(w, "gemm_ce_weighted");
  if (rc != DB200_OK) return rc;
  return gemm_run(stream, A, a_mn_major, lda, B, b_mn_major, ldb, D, ldd, M, N, K, epi, nullptr, w);
}

extern "C" int db200_gemm_bf16_gelu(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda, const void* B,
                                    int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M, int N, int K,
                                    const db200_gemm_epilogue* epi, void* z, int64_t ldz) {
  DB200_REQUIRE(epi != nullptr && epi->mode == DB200_EPI_STORE, DB200_E_INVALID,
                "gemm_gelu: needs an epilogue descriptor with mode DB200_EPI_STORE");
  DB200_REQUIRE(!epi->out_f32 && !epi->relu && !epi->residual, DB200_E_INVALID,
                "gemm_gelu: bf16 output only, without relu or a residual");
  if (z) DB200_REQUIRE(aligned16(z) && ldz % 8 == 0 && ldz >= N, DB200_E_ALIGN,
                       "gemm_gelu: z must be 16-byte aligned with ldz %% 8 == 0 and ldz >= N (got ldz=%lld)",
                       (long long)ldz);
  return gemm_run(stream, A, a_mn_major, lda, B, b_mn_major, ldb, D, ldd, M, N, K, epi, nullptr, nullptr, G_GELU_FWD,
                  z, z ? ldz : 0);
}

extern "C" int db200_gemm_bf16_gelu_bwd(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda,
                                        const void* B, int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M, int N,
                                        int K, const db200_gemm_epilogue* epi) {
  DB200_REQUIRE(epi != nullptr && epi->mode == DB200_EPI_RELU_BWD, DB200_E_INVALID,
                "gemm_gelu_bwd: needs an epilogue descriptor with mode DB200_EPI_RELU_BWD (aux = z)");
  return gemm_run(stream, A, a_mn_major, lda, B, b_mn_major, ldb, D, ldd, M, N, K, epi, nullptr, nullptr, G_GELU_BWD);
}

// the gated MLP: act 0 = ReGLU, 1 = GEGLU (DB200_ACT_*); N = the h width, a multiple of 64
static int glu_check(const void* A, const void* B, const void* D, int N, int act, const char* fn) {
  DB200_REQUIRE(act == DB200_ACT_RELU || act == DB200_ACT_GELU, DB200_E_INVALID,
                "%s: act must be DB200_ACT_RELU or DB200_ACT_GELU (got %d)", fn, act);
  DB200_REQUIRE(A && B && D, DB200_E_INVALID, "%s: NULL operand or output", fn);
  DB200_REQUIRE(N > 0 && N % 64 == 0, DB200_E_INVALID, "%s: N must be a positive multiple of 64 (got %d)", fn, N);
  return DB200_OK;
}

extern "C" int db200_gemm_bf16_glu(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda, const void* B,
                                   int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M, int N, int K,
                                   const db200_gemm_epilogue* epi, int act, void* z, int64_t ldz) {
  DB200_REQUIRE(epi != nullptr && epi->mode == DB200_EPI_STORE, DB200_E_INVALID,
                "gemm_glu: needs an epilogue descriptor with mode DB200_EPI_STORE");
  DB200_REQUIRE(!epi->out_f32 && !epi->relu && !epi->residual, DB200_E_INVALID,
                "gemm_glu: bf16 output only, without relu or a residual");
  const int rc = glu_check(A, B, D, N, act, "gemm_glu");
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(!a_mn_major && b_mn_major, DB200_E_UNSUPPORTED, "gemm_glu: needs a k-major A and an mn-major B");
  DB200_REQUIRE(ldb >= 2 * (int64_t)N, DB200_E_INVALID,
                "gemm_glu: B holds the value and gate columns: ldb must be >= 2N (got ldb=%lld, N=%d)", (long long)ldb, N);
  if (z) DB200_REQUIRE(aligned16(z) && ldz % 8 == 0 && ldz >= 2 * (int64_t)N, DB200_E_ALIGN,
                       "gemm_glu: z must be 16-byte aligned with ldz %% 8 == 0 and ldz >= 2N (got ldz=%lld, N=%d)",
                       (long long)ldz, N);
  return gemm_run(stream, A, a_mn_major, lda, B, b_mn_major, ldb, D, ldd, M, N, K, epi, nullptr, nullptr,
                  act == DB200_ACT_GELU ? G_GLU_GELU_FWD : G_GLU_RELU_FWD, z, z ? ldz : 0);
}

extern "C" int db200_gemm_bf16_glu_bwd(db200_stream_t stream, const void* A, int a_mn_major, int64_t lda,
                                       const void* B, int b_mn_major, int64_t ldb, void* D, int64_t ldd, int M, int N,
                                       int K, const db200_gemm_epilogue* epi, int act) {
  DB200_REQUIRE(epi != nullptr && epi->mode == DB200_EPI_RELU_BWD, DB200_E_INVALID,
                "gemm_glu_bwd: needs an epilogue descriptor with mode DB200_EPI_RELU_BWD (aux = z)");
  const int rc = glu_check(A, B, D, N, act, "gemm_glu_bwd");
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(!a_mn_major && !b_mn_major, DB200_E_UNSUPPORTED, "gemm_glu_bwd: needs k-major A and B");
  DB200_REQUIRE(ldd >= 2 * (int64_t)N, DB200_E_INVALID,
                "gemm_glu_bwd: D is [M][2N] (dzv | dzg): ldd must be >= 2N (got ldd=%lld, N=%d)", (long long)ldd, N);
  DB200_REQUIRE(epi->aux && aligned16(epi->aux) && epi->ldaux % 8 == 0 && epi->ldaux >= 2 * (int64_t)N, DB200_E_ALIGN,
                "gemm_glu_bwd: aux = z [M][2N] must be 16-byte aligned with ldaux %% 8 == 0 and ldaux >= 2N (got %lld)",
                (long long)epi->ldaux);
  return gemm_run(stream, A, a_mn_major, lda, B, b_mn_major, ldb, D, ldd, M, N, K, epi, nullptr, nullptr,
                  act == DB200_ACT_GELU ? G_GLU_GELU_BWD : G_GLU_RELU_BWD);
}
