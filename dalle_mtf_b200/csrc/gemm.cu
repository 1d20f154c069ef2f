// K3/K5/K6/K7/K8 — persistent, warp-specialised bf16 GEMM on wgmma for sm_90a.
//
//   D[M,N] = A[M,K] * B[K,N],  fp32 accumulation in registers, operands staged in shared memory by TMA (128B swizzle).
//
//   warp 0    : TMA producer (one elected lane)            smem ring: STAGES x {A 128x64, B BNx64} bf16
//   warps 1-3 : idle
//   warps 4-11: two consumer warpgroups.  Warpgroup g issues wgmma m64 x BN x 16 for rows [64g, 64g+64) of the tile;
//               at the end of a tile both write their accumulators to a shared-memory tile, and the 8 warps run the
//               epilogue on it (each accumulator row split between two threads) -> bias / ReLU / residual / split-K
//               reduction / cross-entropy statistics and gradient.  The producer keeps loading the next tile meanwhile.
//
// Either operand may be K-major or MN-major in global memory; the tensor maps and the wgmma descriptors absorb the
// difference, so forward (x*W), dgrad (dy*W^T) and wgrad (x^T*dy) are the same kernel.
//
// Reference call sites replaced: every mtf einsum / mtf.layers.dense of src/dalle_mtf/models.py (235-244, 303-311,
// 317-324, 361-371, 391-395) and their gradients produced by mtf.gradients (src/optimizers.py:34).
#include "gemm_common.cuh"
#include "wgmma.cuh"

namespace db200 {

// BN = 128: the 128 x 128 fp32 accumulator tile (64 KiB) and four 32 KiB stages fit the 227 KiB of an H100 SM.
constexpr int GBN = 128;
constexpr int G_STAGES = 4;
constexpr uint32_t G_B_BYTES = GBN * BK * 2;
constexpr uint32_t G_STAGE_BYTES = A_BYTES + G_B_BYTES;
constexpr uint32_t G_ACC_BYTES = BM * GBN * 4;
constexpr size_t G_SMEM_BYTES =
    1024 /*align slack*/ + G_ACC_BYTES + size_t(G_STAGES) * G_STAGE_BYTES + 256 /*barriers*/ + 8 * 4096 /*staging*/;
static_assert(G_SMEM_BYTES <= 227 * 1024, "GEMM shared memory exceeds the H100 per-block limit");

template <int TA, int TB>  // operand majors (1 = MN-major), compile-time for wgmma
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
  const uint32_t stg_base = bars + 256;             // 8 x STG_BYTES, 16-byte aligned

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(full_bar + 8 * i, 1);
      mbar_init(empty_bar + 8 * i, 2);  // one arrive per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int total_tiles = p.m_tiles * p.n_tiles * p.splits;

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    // converged warp, issuer picked by elect.sync: TMA instructions compile to plain uniform-datapath code
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int m0 = t.m_blk * BM, n0 = t.n_blk * BN;
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
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ consumers: MMA, then epilogue
    const int ew = warp - 4;
    const int wg = ew >> 2;        // consumer warpgroup: accumulator rows [64 wg, 64 wg + 64)
    const int wq = ew & 3;         // epilogue: rows [32 wq, 32 wq + 32) ...
    const int half = ew >> 2;      // ... and columns [half * BN/2, (half + 1) * BN/2)
    constexpr int CH = BN / 64;    // 32-column chunks per half
    const uint32_t stg = stg_base + ew * STG_BYTES;
    // K-major: a K-step advances 16 elements (32 B) inside the 128 B swizzle row and warpgroup g starts 64 rows (8 KiB)
    // in; MN-major: a K-step is 16 k-rows (2 KiB) and warpgroup g takes the g-th 64-wide slab (SLAB_BYTES apart).
    constexpr uint64_t astep = TA ? 128u : 2u, bstep = TB ? 128u : 2u;
    const uint32_t a_wg = wg * (TA ? SLAB_BYTES : 64u * 128u);
    float d[BN / 2];
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile);
      const int row0 = t.m_blk * BM + wq * 32;
      const int row = row0 + lane;
      const bool row_ok = row < p.M;
      const int cbase = t.n_blk * BN + half * (BN / 2);
      // pull this half-tile's bias into L1 and the per-element operands (ReLU mask / residual rows) into L2 while
      // the accumulator is being produced
      if (p.bias && lane < BN / 64 && cbase + lane * 32 < p.N)
        asm volatile("prefetch.global.L1 [%0];" ::"l"(p.bias + cbase + lane * 32));
      if (row_ok && cbase < p.N) {
        if (p.aux) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.aux + (long long)row * p.ldaux + cbase));
        if (p.residual) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.residual + (long long)row * p.ldr + cbase));
      }
      uint32_t prev_stage = 0;
      // zero the accumulator here rather than through wgmma's scale-d: its registers are then dead between the
      // shared-memory store of one tile and the start of the next (no spill around the epilogue)
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
      named_bar_sync(1, 256);  // the previous tile's epilogue has finished reading the accumulator tile
      acc_store_smem<BN>(d, sAcc >> 2, 64 * wg);
      named_bar_sync(1, 256);
      const uint32_t t_addr = (sAcc >> 2) + (wq * 32 + lane) * BN + half * (BN / 2);
      switch (p.mode) {
        case DB200_EPI_STORE:    epi_store<CH>(p, t_addr, row, row_ok, cbase, stg, row0, lane); break;
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
  }
}

template <int TA, int TB>
static int launch_gemm(cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p) {
  static const cudaError_t attr_rc = cudaFuncSetAttribute(gemm_tc_kernel<TA, TB>,
                                                          cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                          (int)G_SMEM_BYTES);  // once, thread-safe (magic static)
  DB200_CUDA(attr_rc);
  const int total = p.m_tiles * p.n_tiles * p.splits;
  const int grid = total < sm_count() ? total : sm_count();
  gemm_tc_kernel<TA, TB><<<grid, GEMM_THREADS, G_SMEM_BYTES, stream>>>(tmA, tmB, p);
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
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(epi != nullptr, DB200_E_INVALID, "gemm: epilogue descriptor is NULL");
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
    DB200_REQUIRE(epi->labels && epi->lse && epi->n_valid > 0 && epi->n_valid <= N && epi->alpha > 0.f,
                  DB200_E_INVALID, "gemm: CE_GRAD needs labels/lse, 0 < n_valid <= N and alpha > 0");
  DB200_REQUIRE(mode == DB200_EPI_ATOMIC || epi->split_k <= 1, DB200_E_INVALID,
                "gemm: split_k > 1 is only valid with DB200_EPI_ATOMIC");
  const int splits = gemm_splits(M, N, K, epi);
  const int kb_total = (K + BK - 1) / BK;
  DB200_REQUIRE(workspace_ok(epi->workspace, epi->workspace_bytes, db200_gemm_workspace_bytes(M, N, K, epi)),
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

  p.n_tiles = (N + GBN - 1) / GBN;
  p.n_parts = 2 * p.n_tiles;

  // MN-major operands whose MN extent is a multiple of 64: one rank-3 map {64, K, MN/64} (stride of the slab index =
  // 128 bytes) fetches every 64-wide slab of a stage with a single TMA instruction instead of one per slab.
  p.a_3d = (p.a_mn && M % 64 == 0) ? 1 : 0;
  p.b_3d = (p.b_mn && N % 64 == 0) ? 1 : 0;
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
  } else if (p.b_mn) rc = make_tmap_2d(&tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, 64, BK);
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
  if (p.a_mn) rc = p.b_mn ? launch_gemm<1, 1>(stream, tmA, tmB, p) : launch_gemm<1, 0>(stream, tmA, tmB, p);
  else        rc = p.b_mn ? launch_gemm<0, 1>(stream, tmA, tmB, p) : launch_gemm<0, 0>(stream, tmA, tmB, p);
  if (rc != DB200_OK) return rc;
  if (p.splits > 1) return reduce_splits_add(stream, static_cast<const float*>(p.D), p.splits, M, N, d_out, ldd);
  if (colsum_out) return reduce_rows_add(stream, p.colsum, row_blocks, N, colsum_out);
  return DB200_OK;
}
