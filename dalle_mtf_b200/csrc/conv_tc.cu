// K11 (tensor-core path) — NHWC bf16 convolutions as im2col-free implicit GEMMs on wgmma.
//
// (1) gather-GEMM  (forward conv, forward conv-transpose, every dgrad):
//        y[pix, n] = epi( sum_{tap} sum_k  x[src(pix, tap), k] * W_tap[k][n] )
//     M = output pixels (tile = TN x TH x TW = 128 pixels), N = produced channels, K = taps x contracted channels.
//     One k-block is (one filter tap, 64 channels): its A operand is ONE 4-D TMA box {64 ch, TW, TH, TN} of the
//     gathered tensor shifted by the tap offset — out-of-image coordinates are zero-filled by TMA, which IS the SAME
//     padding — landing in smem as a [128 pixels][64 ch] 128B-swizzled K-major tile.  The B operand is a slab of
//     the bf16 kernel, K-major or MN-major depending on which index of the 4-D kernel is contracted.  Strided
//     gathers use four parity views of the tensor (so every tap is again a dense box); strided scatters (conv-transpose
//     forward, stride-2 dgrad) run one launch per output parity.  No im2col buffer exists in HBM or smem.
// (2) wgrad:  dW_tap[a][b] += sum_pix P[src(pix,tap), a] * Q[src'(pix,tap), b]
//     M = a (channels of P), N = b (channels of Q), K = pixels: both operands are the same 4-D TMA boxes used as
//     MN-major wgmma operands (k rows = pixels); split over pixels, fp32 accumulation in registers, red.add into dW.
//
// Same warp-specialised pipeline as gemm.cu (TMA producer warp / two wgmma consumer warpgroups whose accumulators go
// through a shared-memory tile to the 8-warp epilogue).
// Reference: tf.layers.conv2d / conv2d_transpose call sites src/vae_tf/models.py:95-109, 139-155 and their gradients.
#include "gemm_common.cuh"  // staging helpers for coalesced epilogue I/O
#include "wgmma.cuh"

namespace db200 {

constexpr int CT_THREADS = 384;
constexpr uint32_t CT_A_BYTES = 128 * 64 * 2;
constexpr uint32_t CT_SLAB = 64 * 128;

template <int BN>
struct ConvTcCfg {
  static_assert(BN == 64 || BN == 128, "wgmma tile width");
  static constexpr int STAGES = 4;
  static constexpr uint32_t B_BYTES = BN * 64 * 2;
  static constexpr uint32_t STAGE_BYTES = CT_A_BYTES + B_BYTES;
  static constexpr uint32_t ACC_BYTES = 128 * BN * 4;  // fp32 accumulator tile
  static constexpr size_t SMEM_BYTES =
      1024 + ACC_BYTES + size_t(STAGES) * STAGE_BYTES + 256 + 8 * 4096 /*epilogue staging*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "conv shared memory exceeds the H100 per-block limit");
};

struct ConvTcTap {
  int dy, dx, map;  // coordinate offsets inside gathered-tensor view `map`
  int wrow;         // first row of this tap's slab in the 2-D weight matrix
};

struct ConvTcParams {
  int NB, OH, OW;          // enumeration grid of output pixels
  int out_H, out_W;        // spatial dims of the output tensor
  int out_stride, oa, ob;  // output pixel = (oy*out_stride + oa, ox*out_stride + ob)
  int K, Nn;               // contracted / produced channels
  int TW, TH, TN;
  int tiles_w, tiles_h, tiles_n, tiles_c;
  int ntaps, kchunks;
  int b_kmajor;            // 1: weight matrix rows = produced channel, K contiguous;  0: rows = k, N contiguous
  int b_3d;                // MN-major weight slabs fetched by ONE rank-3 TMA op {64, rows, Nn/64}
  ConvTcTap taps[16];
  int relu;
  const float* bias;
  const bf16* residual;    // same layout as y
  const bf16* mask;        // same layout as y: y = mask > 0 ? y : 0   (ReLU backward)
  bf16* y;
};

struct ConvTile {
  int n0, oy0, ox0, c_blk;
};
__device__ __forceinline__ ConvTile conv_decode(const ConvTcParams& p, int tile) {
  ConvTile t;
  t.c_blk = tile % p.tiles_c; tile /= p.tiles_c;   // channel tiles innermost: neighbours share the A box (L2)
  t.ox0 = (tile % p.tiles_w) * p.TW; tile /= p.tiles_w;
  t.oy0 = (tile % p.tiles_h) * p.TH; tile /= p.tiles_h;
  t.n0 = tile * p.TN;
  return t;
}

template <int BN>
__global__ void __launch_bounds__(CT_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
               const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmA3,
               const __grid_constant__ CUtensorMap tmB, const ConvTcParams p) {
  using Cfg = ConvTcCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t sAcc = base;
  const uint32_t sA = base + Cfg::ACC_BYTES;
  const uint32_t sB = sA + STAGES * CT_A_BYTES;
  const uint32_t bars = sA + STAGES * Cfg::STAGE_BYTES;
  const uint32_t full_bar = bars, empty_bar = bars + 8 * STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA0);
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

  const int total_tiles = p.tiles_n * p.tiles_h * p.tiles_w * p.tiles_c;
  const int nkb = p.ntaps * p.kchunks;

  if (warp == 0) {
    // converged producer warp; elect.sync picks the lane that issues the TMA instructions (uniform-datapath code, no
    // per-lane waterfall around each UTMALDG)
    {
      const CUtensorMap* maps[4] = {&tmA0, &tmA1, &tmA2, &tmA3};
      uint32_t stage = 0, phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const ConvTile t = conv_decode(p, tile);
        for (int tap = 0; tap < p.ntaps; ++tap) {
          const ConvTcTap tp = p.taps[tap];
          for (int kc = 0; kc < p.kchunks; ++kc) {
            mbar_wait_mma(empty_bar + 8 * stage, phase ^ 1);
            const uint32_t fb = full_bar + 8 * stage;
            if (elect_one_sync()) {
            mbar_expect_tx(fb, Cfg::STAGE_BYTES);
            tma_load_4d(sA + stage * CT_A_BYTES, maps[tp.map], fb, kc * 64, t.ox0 + tp.dx, t.oy0 + tp.dy, t.n0);
            const uint32_t b_dst = sB + stage * Cfg::B_BYTES;
            if (p.b_kmajor) {
              tma_load_2d(b_dst, &tmB, fb, kc * 64, tp.wrow + t.c_blk * BN);
            } else if (p.b_3d) {
              tma_load_3d(b_dst, &tmB, fb, 0, tp.wrow + kc * 64, (t.c_blk * BN) >> 6);
            } else {
#pragma unroll
              for (int s = 0; s < BN / 64; ++s)
                tma_load_2d(b_dst + s * CT_SLAB, &tmB, fb, t.c_blk * BN + 64 * s, tp.wrow + kc * 64);
            }
            }  // elect
            __syncwarp();
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // Consumers: warpgroup g computes accumulator rows (pixels) [64 g, 64 g + 64) with wgmma, then all 8 warps run the
    // epilogue from the shared-memory accumulator tile.  A thread owns one output PIXEL (accumulator row) and its
    // channels are contiguous in NHWC, so the same coalescing scheme as the GEMM applies: 32 pixels x 64 channels are
    // transposed through a swizzled 4 KiB smem block and every global access covers 4 pixels x 128 contiguous bytes
    // (outputs, residual and ReLU-mask operands).
    const int ew = warp - 4, wq = ew & 3, half = ew >> 2, wg = ew >> 2;
    constexpr int HALF = BN / 2;
    const uint32_t stg = bars + 256 + ew * STG_BYTES;
    const int slot = lane & 7, rsub = lane >> 3;
    const uint64_t bstep = p.b_kmajor ? 2u : 128u;      // (32 B | 2 KiB) >> 4 per 16-deep K-step
    float d[BN / 2];
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const ConvTile t = conv_decode(p, tile);
      uint32_t prev_stage = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait_mma(full_bar + 8 * stage, phase);
        const uint32_t a_base = sA + stage * CT_A_BYTES + wg * (64u * 128u), b_base = sB + stage * Cfg::B_BYTES;
        const uint64_t ad0 = smem_desc_sw128(a_base, 0, 1024);
        const uint64_t bd0 = smem_desc_sw128(b_base, p.b_kmajor ? 0u : CT_SLAB, 1024);
        wgmma_fence();
        if (p.b_kmajor) {
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_m64<BN, 0, 0>(d, ad0 + 2u * k, bd0 + bstep * k, (kb > 0 || k > 0) ? 1u : 0u);
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_m64<BN, 0, 1>(d, ad0 + 2u * k, bd0 + bstep * k, (kb > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(empty_bar + 8 * prev_stage);
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(empty_bar + 8 * prev_stage);
      // element offsets (or -1) of the 8 pixels this lane moves during block loads / stores
      long long poff[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = wq * 32 + i * 4 + rsub;
        const int tw = r % p.TW, th = (r / p.TW) % p.TH, tn = r / (p.TW * p.TH);
        const int n = t.n0 + tn, oy = t.oy0 + th, ox = t.ox0 + tw;
        poff[i] = (n < p.NB && oy < p.OH && ox < p.OW)
                      ? (((long long)n * p.out_H + (oy * p.out_stride + p.oa)) * p.out_W + (ox * p.out_stride + p.ob)) * p.Nn
                      : -1;
      }
      named_bar_sync(1, 256);  // the previous tile's epilogue is done with the accumulator tile
      acc_store_smem<BN>(d, sAcc >> 2, 64 * wg);
      named_bar_sync(1, 256);
      const uint32_t t_addr = (sAcc >> 2) + (wq * 32 + lane) * BN + half * HALF;
      const int cbase = t.c_blk * BN + half * HALF;
      constexpr int CW = (HALF >= 64) ? 64 : 32;  // channels per staged block
#pragma unroll 1
      for (int cb = 0; cb < HALF / CW; ++cb) {
        const int colp = cbase + cb * CW;
        if (colp >= p.Nn) break;
        float v[CW];
#pragma unroll
        for (int h = 0; h < CW / 32; ++h) {
          uint32_t rr[32];
          acc_ld_x32(t_addr + cb * CW + h * 32, rr);
#pragma unroll
          for (int j = 0; j < 32; ++j) v[h * 32 + j] = __uint_as_float(rr[j]);
        }
        if (p.bias) {
#pragma unroll
          for (int g = 0; g < CW / 8; ++g) {
            if (colp + g * 8 + 8 > p.Nn) break;
            float bb[8];
            load8(p.bias + colp + g * 8, bb);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[g * 8 + j] += bb[j];
          }
        }
        if (p.relu) {
#pragma unroll
          for (int j = 0; j < CW; ++j) v[j] = fmaxf(v[j], 0.f);
        }
        // optional operands with the output's layout: block-load -> per-row read
        for (int which = 0; which < 2; ++which) {
          const bf16* src = which == 0 ? p.mask : p.residual;
          if (!src) continue;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int col = colp + slot * 8;
            uint4 q = make_uint4(0, 0, 0, 0);
            if (poff[i] >= 0 && slot * 8 < CW && col + 8 <= p.Nn) q = __ldg(reinterpret_cast<const uint4*>(src + poff[i] + col));
            st_shared_v4u(stg_addr(stg, i * 4 + rsub, slot), q.x, q.y, q.z, q.w);
          }
          __syncwarp();
#pragma unroll
          for (int h = 0; h < CW / 32; ++h) {
            float o[32];
            stage_get_bf16(stg, lane, h, o);
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              if (which == 0) v[h * 32 + j] = o[j] > 0.f ? v[h * 32 + j] : 0.f;
              else            v[h * 32 + j] += o[j];
            }
          }
          __syncwarp();
        }
#pragma unroll
        for (int h = 0; h < CW / 32; ++h) stage_put_bf16(stg, lane, h, v + h * 32);
        __syncwarp();
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int col = colp + slot * 8;
          const uint4 q = ld_shared_v4u(stg_addr(stg, i * 4 + rsub, slot));
          if (poff[i] >= 0 && slot * 8 < CW && col + 8 <= p.Nn) *reinterpret_cast<uint4*>(p.y + poff[i] + col) = q;
        }
        __syncwarp();
      }
    }
  }
}

template <int BN>
static int conv_tc_launch(cudaStream_t stream, const CUtensorMap* tmA, const CUtensorMap& tmB, const ConvTcParams& p) {
  using Cfg = ConvTcCfg<BN>;
  static const cudaError_t attr_rc = cudaFuncSetAttribute(conv_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM_BYTES);  // once, thread-safe
  DB200_CUDA(attr_rc);
  const int total = p.tiles_n * p.tiles_h * p.tiles_w * p.tiles_c;
  const int grid = total < sm_count() ? total : sm_count();
  conv_tc_kernel<BN><<<grid, CT_THREADS, Cfg::SMEM_BYTES, stream>>>(tmA[0], tmA[1], tmA[2], tmA[3], tmB, p);
  return check_launch("conv_tc_kernel");
}

static int pow2_floor(int x) {
  int p = 1;
  while (p * 2 <= x) p *= 2;
  return p;
}

// 4-D maps of an NHWC bf16 tensor [N][H][W][C]: the plain view (stride 1) or the four parity views
// view(ph,pw)[n][h2][w2][c] = t[n][2*h2+ph][2*w2+pw][c]   (H, W even).
// slabs > 0: rank-5 variant {64, W, H, N, C/64} with a box of `slabs` 64-channel slabs (C % 64 == 0).
static int make_act_maps(CUtensorMap* tm, const bf16* t, int N, int H, int W, int C, int stride, const uint32_t* box,
                         int slabs = 0) {
  int rc;
  if (slabs > 0) {
    for (int ph = 0; ph < (stride == 1 ? 1 : 2); ++ph)
      for (int pw = 0; pw < (stride == 1 ? 1 : 2); ++pw) {
        const uint64_t s = (uint64_t)stride;
        uint64_t dims[5] = {64, (uint64_t)W / s, (uint64_t)H / s, (uint64_t)N, (uint64_t)C / 64};
        uint64_t str[4] = {s * C * 2, s * W * C * 2, (uint64_t)H * W * C * 2, 128};
        uint32_t bx[5] = {64, box[1], box[2], box[3], (uint32_t)slabs};
        rc = make_tmap_bf16(&tm[ph * 2 + pw], t + ((long long)ph * W + pw) * C, 5, dims, str, bx);
        if (rc != DB200_OK) return rc;
      }
    if (stride == 1) tm[1] = tm[2] = tm[3] = tm[0];
    return DB200_OK;
  }
  if (stride == 1) {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t str[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
    rc = make_tmap_bf16(&tm[0], t, 4, dims, str, box);
    if (rc != DB200_OK) return rc;
    tm[1] = tm[2] = tm[3] = tm[0];
    return DB200_OK;
  }
  for (int ph = 0; ph < 2; ++ph)
    for (int pw = 0; pw < 2; ++pw) {
      uint64_t dims[4] = {(uint64_t)C, (uint64_t)W / 2, (uint64_t)H / 2, (uint64_t)N};
      uint64_t str[3] = {(uint64_t)2 * C * 2, (uint64_t)2 * W * C * 2, (uint64_t)H * W * C * 2};
      rc = make_tmap_bf16(&tm[ph * 2 + pw], t + ((long long)ph * W + pw) * C, 4, dims, str, box);
      if (rc != DB200_OK) return rc;
    }
  return DB200_OK;
}

static void choose_tile(int OW, int OH, int& TW, int& TH, int& TN) {
  TW = pow2_floor(OW < 16 ? OW : 16);
  const int th = 128 / TW;
  TH = pow2_floor(OH < th ? OH : th);
  TN = 128 / (TW * TH);
}

// offset e (in full-resolution pixels) -> (parity, coordinate offset in the parity view)
static void split_parity(int e, int& par, int& d) {
  par = ((e % 2) + 2) % 2;
  d = (e - par) / 2;
}

static int run_gather(cudaStream_t stream, ConvTcParams& p, const CUtensorMap* tmA, const void* w_bf16, int wrows) {
  choose_tile(p.OW, p.OH, p.TW, p.TH, p.TN);
  p.tiles_w = (p.OW + p.TW - 1) / p.TW;
  p.tiles_h = (p.OH + p.TH - 1) / p.TH;
  p.tiles_n = (p.NB + p.TN - 1) / p.TN;
  p.kchunks = p.K / 64;
  const int bn = p.Nn >= 128 ? 128 : 64;
  p.tiles_c = (p.Nn + bn - 1) / bn;
  CUtensorMap tmB;
  int rc;
  p.b_3d = (!p.b_kmajor && p.Nn % 64 == 0) ? 1 : 0;
  if (p.b_kmajor) rc = make_tmap_2d(&tmB, w_bf16, (uint64_t)p.K, (uint64_t)wrows, (uint64_t)p.K, 64, (uint32_t)bn);
  else if (p.b_3d) {
    uint64_t dims[3] = {64, (uint64_t)wrows, (uint64_t)p.Nn / 64};
    uint64_t str[2] = {(uint64_t)p.Nn * 2, 128};
    uint32_t box[3] = {64, 64, (uint32_t)bn / 64};
    rc = make_tmap_bf16(&tmB, w_bf16, 3, dims, str, box);
  } else rc = make_tmap_2d(&tmB, w_bf16, (uint64_t)p.Nn, (uint64_t)wrows, (uint64_t)p.Nn, 64, 64);
  if (rc != DB200_OK) return rc;
  if (bn == 128) return conv_tc_launch<128>(stream, tmA, tmB, p);
  return conv_tc_launch<64>(stream, tmA, tmB, p);
}

// ------------------------------------------------------------------------------------------------------------------
// wgrad on wgmma
// ------------------------------------------------------------------------------------------------------------------
struct WgradTcTap {
  int pmap, pdy, pdx, qmap, qdy, qdx;
  long long w_off;
};
struct WgradTcParams {
  int NB, OH, OW;  // enumeration grid (the contracted pixels)
  int TW, TH, TN, tiles_w, tiles_h, tiles_n;
  int pC, qC;      // channels of P (M) and Q (N)
  int a_tiles, b_tiles, ntaps, splits;
  long long a_stride, b_stride;
  WgradTcTap taps[16];
  float* dw;
};

template <int BN>
struct WgradCfg {
  static_assert(BN == 64 || BN == 128, "wgmma tile width");
  static constexpr int STAGES = (BN == 128) ? 2 : 3;
  static constexpr uint32_t A_BYTES = 2 * 128 * 128;         // two 64-channel slabs of [128 pixels][64 ch]
  static constexpr uint32_t B_BYTES = (BN / 64) * 128 * 128;
  static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr uint32_t ACC_BYTES = 128 * BN * 4;        // fp32 accumulator tile
  static constexpr size_t SMEM_BYTES = 1024 + ACC_BYTES + size_t(STAGES) * STAGE_BYTES + 256;
  static_assert(SMEM_BYTES <= 227 * 1024, "wgrad shared memory exceeds the H100 per-block limit");
};

template <int BN>
__global__ void __launch_bounds__(CT_THREADS, 1)
conv_wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmP0, const __grid_constant__ CUtensorMap tmP1,
                     const __grid_constant__ CUtensorMap tmP2, const __grid_constant__ CUtensorMap tmP3,
                     const __grid_constant__ CUtensorMap tmQ0, const __grid_constant__ CUtensorMap tmQ1,
                     const __grid_constant__ CUtensorMap tmQ2, const __grid_constant__ CUtensorMap tmQ3,
                     const WgradTcParams p) {
  using Cfg = WgradCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t sAcc = base;
  const uint32_t sA = base + Cfg::ACC_BYTES;
  const uint32_t sB = sA + STAGES * Cfg::A_BYTES;
  const uint32_t bars = sA + STAGES * Cfg::STAGE_BYTES;
  const uint32_t full_bar = bars, empty_bar = bars + 8 * STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // work item: (tap, a tile, b tile, pixel split)
  int w = blockIdx.x;
  const int b_blk = w % p.b_tiles; w /= p.b_tiles;
  const int a_blk = w % p.a_tiles; w /= p.a_tiles;
  const int tap_i = w % p.ntaps;
  const int split = w / p.ntaps;
  const WgradTcTap tp = p.taps[tap_i];
  const int total_ptiles = p.tiles_n * p.tiles_h * p.tiles_w;
  const int per = (total_ptiles + p.splits - 1) / p.splits;
  const int pt0 = split * per, pt1 = min(total_ptiles, pt0 + per);

  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(full_bar + 8 * i, 1);
      mbar_init(empty_bar + 8 * i, 2);  // one arrive per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (pt1 > pt0) {
    if (warp == 0) {
      {
        const CUtensorMap* pm[4] = {&tmP0, &tmP1, &tmP2, &tmP3};
        const CUtensorMap* qm[4] = {&tmQ0, &tmQ1, &tmQ2, &tmQ3};
        uint32_t stage = 0, phase = 0;
        for (int pt = pt0; pt < pt1; ++pt) {
          int t = pt;
          const int ox0 = (t % p.tiles_w) * p.TW; t /= p.tiles_w;
          const int oy0 = (t % p.tiles_h) * p.TH; t /= p.tiles_h;
          const int n0 = t * p.TN;
          mbar_wait_mma(empty_bar + 8 * stage, phase ^ 1);
          const uint32_t fb = full_bar + 8 * stage;
          const uint32_t a_dst = sA + stage * Cfg::A_BYTES, b_dst = sB + stage * Cfg::B_BYTES;
          if (elect_one_sync()) {
            mbar_expect_tx(fb, Cfg::STAGE_BYTES);
            // rank-5 maps {64 ch, W, H, N, C/64}: all 64-channel slabs of the operand in one TMA op
            tma_load_5d(a_dst, pm[tp.pmap], fb, 0, ox0 + tp.pdx, oy0 + tp.pdy, n0, a_blk * 2);
            tma_load_5d(b_dst, qm[tp.qmap], fb, 0, ox0 + tp.qdx, oy0 + tp.qdy, n0, b_blk * (BN / 64));
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    } else if (warp >= 4) {
      // consumers: warpgroup g owns accumulator rows [64 g, 64 g + 64) = the g-th 64-channel slab of P
      const int ew = warp - 4, wq = ew & 3, half = ew >> 2, wg = ew >> 2;
      constexpr int HALF = BN / 2;
      float d[BN / 2];
      uint32_t stage = 0, phase = 0, prev_stage = 0;
      for (int pt = pt0; pt < pt1; ++pt) {
        mbar_wait_mma(full_bar + 8 * stage, phase);
        const uint32_t a_base = sA + stage * Cfg::A_BYTES + wg * (128u * 128u), b_base = sB + stage * Cfg::B_BYTES;
        const uint64_t ad0 = smem_desc_sw128(a_base, 128 * 128, 1024), bd0 = smem_desc_sw128(b_base, 128 * 128, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k)  // 16 pixels (2 KiB) per MMA; 64-channel atoms are 16 KiB apart
          wgmma_m64<BN, 1, 1>(d, ad0 + 128u * k, bd0 + 128u * k, (pt > pt0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (pt > pt0 && (threadIdx.x & 127) == 0) mbar_arrive(empty_bar + 8 * prev_stage);
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      acc_store_smem<BN>(d, sAcc >> 2, 64 * wg);
      named_bar_sync(1, 256);
      const int a = a_blk * 128 + wq * 32 + lane;  // row of the accumulator = channel of P
      float* dst = p.dw + tp.w_off + (long long)a * p.a_stride;
      const uint32_t t_addr = (sAcc >> 2) + (wq * 32 + lane) * BN + half * HALF;
#pragma unroll 1
      for (int c = 0; c < HALF / 32; ++c) {
        const int b0 = b_blk * BN + half * HALF + c * 32;
        if (b0 >= p.qC) break;
        uint32_t r[32];
        acc_ld_x32(t_addr + c * 32, r);
        if (a >= p.pC) continue;
        if (p.b_stride == 1 && b0 + 32 <= p.qC && (((tp.w_off + (long long)a * p.a_stride + b0) & 3) == 0)) {
#pragma unroll
          for (int j = 0; j < 32; j += 4)
            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + b0 + j),
                         "f"(__uint_as_float(r[j])), "f"(__uint_as_float(r[j + 1])), "f"(__uint_as_float(r[j + 2])),
                         "f"(__uint_as_float(r[j + 3]))
                         : "memory");
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (b0 + j < p.qC) atomicAdd(dst + (long long)(b0 + j) * p.b_stride, __uint_as_float(r[j]));
        }
      }
    }
  }
}

template <int BN>
static int wgrad_tc_launch(cudaStream_t stream, const CUtensorMap* tmP, const CUtensorMap* tmQ, const WgradTcParams& p) {
  using Cfg = WgradCfg<BN>;
  static const cudaError_t attr_rc = cudaFuncSetAttribute(conv_wgrad_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM_BYTES);  // once, thread-safe
  DB200_CUDA(attr_rc);
  const int grid = p.b_tiles * p.a_tiles * p.ntaps * p.splits;
  conv_wgrad_tc_kernel<BN><<<grid, CT_THREADS, Cfg::SMEM_BYTES, stream>>>(tmP[0], tmP[1], tmP[2], tmP[3], tmQ[0],
                                                                          tmQ[1], tmQ[2], tmQ[3], p);
  return check_launch("conv_wgrad_tc_kernel");
}

static int same_pad(int in, int out, int k, int s) {
  int total = (out - 1) * s + k - in;
  if (total < 0) total = 0;
  return total / 2;
}

static int tc_validate(const db200_conv_desc* c, const char* who) {
  DB200_REQUIRE(c != nullptr, DB200_E_INVALID, "%s: NULL descriptor", who);
  DB200_REQUIRE(!c->act_f32, DB200_E_UNSUPPORTED, "%s: bf16 activations only", who);
  DB200_REQUIRE(c->KH * c->KW <= 16 && (c->stride == 1 || c->stride == 2), DB200_E_UNSUPPORTED,
                "%s: unsupported kernel size / stride", who);
  if (c->transposed) {
    DB200_REQUIRE(c->KH == 4 && c->KW == 4 && c->stride == 2 && c->Ho == 2 * c->H && c->Wo == 2 * c->W,
                  DB200_E_UNSUPPORTED, "%s: conv2d_transpose is implemented for k=4, s=2, SAME only", who);
  } else {
    DB200_REQUIRE(c->Ho == (c->H + c->stride - 1) / c->stride && c->Wo == (c->W + c->stride - 1) / c->stride,
                  DB200_E_INVALID, "%s: Ho/Wo do not match SAME padding", who);
    DB200_REQUIRE(c->stride == 1 || (c->H % 2 == 0 && c->W % 2 == 0), DB200_E_UNSUPPORTED,
                  "%s: stride 2 needs even H and W", who);
  }
  return DB200_OK;
}

}  // namespace db200

using namespace db200;

// y (bf16 NHWC) = [relu](conv(x bf16 NHWC, w bf16) + bias f32) [+ residual bf16].
//   conv:           w = HWIO [kh][kw][cin][cout] viewed as [(kh*kw*cin)][cout];   needs Cin % 64 == 0, Cout % 8 == 0
//   conv-transpose: w = [kh][kw][cout][cin] viewed as [(kh*kw*cout)][cin];        needs Cin % 64 == 0, Cout % 8 == 0
extern "C" int db200_conv2d_fwd_tc(db200_stream_t stream_, const db200_conv_desc* c, const void* x_bf16,
                                   const void* w_bf16, const float* bias, const void* residual_bf16, void* y_bf16) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = tc_validate(c, "conv2d_fwd_tc");
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(x_bf16 && w_bf16 && y_bf16, DB200_E_INVALID, "conv2d_fwd_tc: NULL argument");
  DB200_REQUIRE(c->Cin % 64 == 0 && c->Cout % 8 == 0, DB200_E_UNSUPPORTED,
                "conv2d_fwd_tc: needs Cin %% 64 == 0 and Cout %% 8 == 0 (got %d, %d)", c->Cin, c->Cout);
  DB200_REQUIRE(aligned16(bias) && aligned16(residual_bf16) && aligned16(y_bf16), DB200_E_ALIGN,
                "conv2d_fwd_tc: unaligned pointer");
  ConvTcParams p{};
  p.K = c->Cin; p.Nn = c->Cout;
  p.relu = c->relu; p.bias = bias; p.mask = nullptr;
  p.residual = reinterpret_cast<const bf16*>(residual_bf16);
  p.y = reinterpret_cast<bf16*>(y_bf16);
  p.out_H = c->Ho; p.out_W = c->Wo;
  const bf16* xb = reinterpret_cast<const bf16*>(x_bf16);
  CUtensorMap tmA[4];
  if (!c->transposed) {
    const int pt = same_pad(c->H, c->Ho, c->KH, c->stride), pl = same_pad(c->W, c->Wo, c->KW, c->stride);
    p.NB = c->N; p.OH = c->Ho; p.OW = c->Wo; p.out_stride = 1; p.oa = 0; p.ob = 0;
    p.ntaps = c->KH * c->KW; p.b_kmajor = 0;
    choose_tile(p.OW, p.OH, p.TW, p.TH, p.TN);
    const uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
    rc = make_act_maps(tmA, xb, c->N, c->H, c->W, c->Cin, c->stride, box);
    if (rc != DB200_OK) return rc;
    for (int kh = 0; kh < c->KH; ++kh)
      for (int kw = 0; kw < c->KW; ++kw) {
        ConvTcTap& t = p.taps[kh * c->KW + kw];
        int ph = 0, pw = 0;
        if (c->stride == 1) { t.dy = kh - pt; t.dx = kw - pl; }
        else { split_parity(kh - pt, ph, t.dy); split_parity(kw - pl, pw, t.dx); }
        t.map = ph * 2 + pw;
        t.wrow = (kh * c->KW + kw) * c->Cin;
      }
    return run_gather(stream, p, tmA, w_bf16, p.ntaps * c->Cin);
  }
  // conv-transpose: y[2i+a, 2j+b, co] = sum over the 2x2 taps of that parity of x[i + dy, j + dx, ci] * w[tap][co][ci]
  p.NB = c->N; p.OH = c->H; p.OW = c->W; p.out_stride = 2; p.b_kmajor = 1;
  choose_tile(p.OW, p.OH, p.TW, p.TH, p.TN);
  const uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
  rc = make_act_maps(tmA, xb, c->N, c->H, c->W, c->Cin, 1, box);
  if (rc != DB200_OK) return rc;
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      p.oa = a; p.ob = b; p.ntaps = 0;
      for (int kh = 0; kh < 4; ++kh) {
        if (((a + 1 - kh) & 1) != 0) continue;
        for (int kw = 0; kw < 4; ++kw) {
          if (((b + 1 - kw) & 1) != 0) continue;
          ConvTcTap& t = p.taps[p.ntaps++];
          t.dy = (a + 1 - kh) / 2; t.dx = (b + 1 - kw) / 2; t.map = 0;
          t.wrow = (kh * 4 + kw) * c->Cout;
        }
      }
      rc = run_gather(stream, p, tmA, w_bf16, 16 * c->Cout);
      if (rc != DB200_OK) return rc;
    }
  return DB200_OK;
}

// dx (bf16) = dgrad(dy bf16, w bf16) [masked by x_mask > 0] [+ dres].   Needs Cout % 64 == 0, Cin % 8 == 0.
extern "C" int db200_conv2d_dgrad_tc(db200_stream_t stream_, const db200_conv_desc* c, const void* dy_bf16,
                                     const void* w_bf16, const void* x_mask_bf16, const void* dres_bf16,
                                     void* dx_bf16) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = tc_validate(c, "conv2d_dgrad_tc");
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(dy_bf16 && w_bf16 && dx_bf16, DB200_E_INVALID, "conv2d_dgrad_tc: NULL argument");
  DB200_REQUIRE(c->Cout % 64 == 0 && c->Cin % 8 == 0, DB200_E_UNSUPPORTED,
                "conv2d_dgrad_tc: needs Cout %% 64 == 0 and Cin %% 8 == 0 (got %d, %d)", c->Cout, c->Cin);
  ConvTcParams p{};
  p.K = c->Cout; p.Nn = c->Cin;
  p.relu = 0; p.bias = nullptr;
  p.mask = reinterpret_cast<const bf16*>(x_mask_bf16);
  p.residual = reinterpret_cast<const bf16*>(dres_bf16);
  p.y = reinterpret_cast<bf16*>(dx_bf16);
  p.out_H = c->H; p.out_W = c->W;
  const bf16* dyb = reinterpret_cast<const bf16*>(dy_bf16);
  CUtensorMap tmA[4];
  if (!c->transposed) {
    const int pt = same_pad(c->H, c->Ho, c->KH, c->stride), pl = same_pad(c->W, c->Wo, c->KW, c->stride);
    p.b_kmajor = 1;  // B(k = co, n = ci) = w[tap][ci][co]: rows (tap, ci), co contiguous
    if (c->stride == 1) {
      p.NB = c->N; p.OH = c->H; p.OW = c->W; p.out_stride = 1; p.oa = 0; p.ob = 0;
      p.ntaps = c->KH * c->KW;
      choose_tile(p.OW, p.OH, p.TW, p.TH, p.TN);
      const uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
      rc = make_act_maps(tmA, dyb, c->N, c->Ho, c->Wo, c->Cout, 1, box);
      if (rc != DB200_OK) return rc;
      for (int kh = 0; kh < c->KH; ++kh)
        for (int kw = 0; kw < c->KW; ++kw) {
          ConvTcTap& t = p.taps[kh * c->KW + kw];
          t.dy = pt - kh; t.dx = pl - kw; t.map = 0;
          t.wrow = (kh * c->KW + kw) * c->Cin;
        }
      return run_gather(stream, p, tmA, w_bf16, p.ntaps * c->Cin);
    }
    // stride 2: input pixel (2i+a, 2j+b) receives from taps with (a + pt - kh) even, from dy[i + (a+pt-kh)/2]
    p.NB = c->N; p.OH = c->H / 2; p.OW = c->W / 2; p.out_stride = 2;
    choose_tile(p.OW, p.OH, p.TW, p.TH, p.TN);
    const uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
    rc = make_act_maps(tmA, dyb, c->N, c->Ho, c->Wo, c->Cout, 1, box);
    if (rc != DB200_OK) return rc;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        p.oa = a; p.ob = b; p.ntaps = 0;
        for (int kh = 0; kh < c->KH; ++kh) {
          if (((a + pt - kh) & 1) != 0) continue;
          for (int kw = 0; kw < c->KW; ++kw) {
            if (((b + pl - kw) & 1) != 0) continue;
            ConvTcTap& t = p.taps[p.ntaps++];
            t.dy = (a + pt - kh) / 2; t.dx = (b + pl - kw) / 2; t.map = 0;
            t.wrow = (kh * c->KW + kw) * c->Cin;
          }
        }
        rc = run_gather(stream, p, tmA, w_bf16, c->KH * c->KW * c->Cin);
        if (rc != DB200_OK) return rc;
      }
    return DB200_OK;
  }
  // transposed forward y[2i-1+kh] += x[i] w[kh][kw][co][ci]  =>  dx[i,ci] = sum dy[2i-1+kh, 2j-1+kw, co] w[tap][co][ci]
  p.NB = c->N; p.OH = c->H; p.OW = c->W; p.out_stride = 1; p.oa = 0; p.ob = 0;
  p.ntaps = 16; p.b_kmajor = 0;  // B(k = co, n = ci): rows (tap, co), ci contiguous
  choose_tile(p.OW, p.OH, p.TW, p.TH, p.TN);
  const uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
  rc = make_act_maps(tmA, dyb, c->N, c->Ho, c->Wo, c->Cout, 2, box);
  if (rc != DB200_OK) return rc;
  for (int kh = 0; kh < 4; ++kh)
    for (int kw = 0; kw < 4; ++kw) {
      ConvTcTap& t = p.taps[kh * 4 + kw];
      int ph, pw;
      split_parity(kh - 1, ph, t.dy);
      split_parity(kw - 1, pw, t.dx);
      t.map = ph * 2 + pw;
      t.wrow = (kh * 4 + kw) * c->Cout;
    }
  return run_gather(stream, p, tmA, w_bf16, 16 * c->Cout);
}

// dw (f32, accumulates) += wgrad(x bf16, dy bf16); dbias is NOT computed here (callers use the column-sum kernel).
// Needs Cin % 64 == 0 and Cout % 64 == 0.
extern "C" int db200_conv2d_wgrad_tc(db200_stream_t stream_, const db200_conv_desc* c, const void* x_bf16,
                                     const void* dy_bf16, float* dw) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = tc_validate(c, "conv2d_wgrad_tc");
  if (rc != DB200_OK) return rc;
  DB200_REQUIRE(x_bf16 && dy_bf16 && dw, DB200_E_INVALID, "conv2d_wgrad_tc: NULL argument");
  DB200_REQUIRE(c->Cin % 64 == 0 && c->Cout % 64 == 0, DB200_E_UNSUPPORTED,
                "conv2d_wgrad_tc: needs Cin %% 64 == 0 and Cout %% 64 == 0 (got %d, %d)", c->Cin, c->Cout);
  WgradTcParams p{};
  p.dw = dw;
  p.pC = c->Cin; p.qC = c->Cout;
  const int wg_bn = p.qC >= 128 ? 128 : 64;
  p.ntaps = c->KH * c->KW;
  const bf16* xb = reinterpret_cast<const bf16*>(x_bf16);
  const bf16* dyb = reinterpret_cast<const bf16*>(dy_bf16);
  CUtensorMap tmP[4], tmQ[4];
  if (!c->transposed) {
    const int pt = same_pad(c->H, c->Ho, c->KH, c->stride), pl = same_pad(c->W, c->Wo, c->KW, c->stride);
    p.NB = c->N; p.OH = c->Ho; p.OW = c->Wo;  // contract over output pixels
    choose_tile(p.OW, p.OH, p.TW, p.TH, p.TN);
    const uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
    rc = make_act_maps(tmP, xb, c->N, c->H, c->W, c->Cin, c->stride, box, 2);
    if (rc != DB200_OK) return rc;
    rc = make_act_maps(tmQ, dyb, c->N, c->Ho, c->Wo, c->Cout, 1, box, wg_bn / 64);
    if (rc != DB200_OK) return rc;
    for (int kh = 0; kh < c->KH; ++kh)
      for (int kw = 0; kw < c->KW; ++kw) {
        WgradTcTap& t = p.taps[kh * c->KW + kw];
        int ph = 0, pw = 0;
        if (c->stride == 1) { t.pdy = kh - pt; t.pdx = kw - pl; }
        else { split_parity(kh - pt, ph, t.pdy); split_parity(kw - pl, pw, t.pdx); }
        t.pmap = ph * 2 + pw;
        t.qmap = 0; t.qdy = 0; t.qdx = 0;
        t.w_off = (long long)(kh * c->KW + kw) * c->Cin * c->Cout;
      }
    p.a_stride = c->Cout; p.b_stride = 1;  // dw[tap][ci][co]
  } else {
    p.NB = c->N; p.OH = c->H; p.OW = c->W;  // contract over input (low-res) pixels
    choose_tile(p.OW, p.OH, p.TW, p.TH, p.TN);
    const uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
    rc = make_act_maps(tmP, xb, c->N, c->H, c->W, c->Cin, 1, box, 2);
    if (rc != DB200_OK) return rc;
    rc = make_act_maps(tmQ, dyb, c->N, c->Ho, c->Wo, c->Cout, 2, box, wg_bn / 64);
    if (rc != DB200_OK) return rc;
    for (int kh = 0; kh < 4; ++kh)
      for (int kw = 0; kw < 4; ++kw) {
        WgradTcTap& t = p.taps[kh * 4 + kw];
        int ph, pw;
        split_parity(kh - 1, ph, t.qdy);
        split_parity(kw - 1, pw, t.qdx);
        t.qmap = ph * 2 + pw;
        t.pmap = 0; t.pdy = 0; t.pdx = 0;
        t.w_off = (long long)(kh * 4 + kw) * c->Cout * c->Cin;
      }
    p.a_stride = 1; p.b_stride = c->Cin;  // dw[tap][co][ci]
  }
  p.tiles_w = (p.OW + p.TW - 1) / p.TW;
  p.tiles_h = (p.OH + p.TH - 1) / p.TH;
  p.tiles_n = (p.NB + p.TN - 1) / p.TN;
  const int bn = wg_bn;
  p.a_tiles = (p.pC + 127) / 128;
  p.b_tiles = (p.qC + bn - 1) / bn;
  const int items = p.a_tiles * p.b_tiles * p.ntaps;
  const int total_ptiles = p.tiles_n * p.tiles_h * p.tiles_w;
  int splits = (sm_count() * 2 + items - 1) / items;
  if (splits > total_ptiles) splits = total_ptiles;
  if (splits < 1) splits = 1;
  const int per = (total_ptiles + splits - 1) / splits;
  p.splits = (total_ptiles + per - 1) / per;  // every split owns at least one pixel tile
  if (bn == 128) return wgrad_tc_launch<128>(stream, tmP, tmQ, p);
  return wgrad_tc_launch<64>(stream, tmP, tmQ, p);
}
