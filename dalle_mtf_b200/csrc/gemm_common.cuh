// GEMM kernel parameters, tile decoding and the epilogue routines that turn the shared-memory accumulator tile
// (wgmma.cuh: acc_store_smem / acc_ld_x32) into global-memory results; the convolutions reuse the staging helpers.
#pragma once
#include "common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace db200 {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int GEMM_THREADS = 384;  // 4 control warps + 2 consumer warpgroups
constexpr int GROUP_M = 8;
constexpr uint32_t SLAB_BYTES = BK * 128;  // one MN-major slab: [BK k-rows][64 bf16] = 8 KiB
constexpr uint32_t A_BYTES = BM * BK * 2;  // 16 KiB

struct GemmParams {
  int M, N, K;
  int a_mn, b_mn;
  int a_3d, b_3d;  // MN-major operand described by ONE rank-3 map {64, K, MN/64}: all slabs of a stage in one TMA op
  int m_tiles, n_tiles, splits, kb_total;
  int mode, out_f32, relu;
  float alpha;
  void* D;
  long long ldd;
  const float* bias;
  const bf16* residual;
  long long ldr;
  const bf16* aux;
  long long ldaux;
  const int* labels;
  float* part_max;
  float* part_sum;
  float* label_logit;
  const float* lse;
  int n_valid;
  int n_parts;  // CE_STATS: partials per row = 2 * n_tiles (one per half tile)
  float* colsum;  // CE_GRAD / RELU_BWD: workspace [M/32 row blocks][N] of column sums (bias gradient), or NULL
};

struct TileCoord {
  int m_blk, n_blk, kb0, kb1, split;
};

__device__ __forceinline__ TileCoord decode_tile(const GemmParams& p, int tile) {
  const int mn_tiles = p.m_tiles * p.n_tiles;
  const int split = tile / mn_tiles;
  const int mn = tile - split * mn_tiles;
  const int group_sz = GROUP_M * p.n_tiles;
  const int group = mn / group_sz;
  const int first_m = group * GROUP_M;
  const int gm = min(GROUP_M, p.m_tiles - first_m);
  const int in_group = mn - group * group_sz;
  TileCoord t;
  t.m_blk = first_m + in_group % gm;
  t.n_blk = in_group / gm;
  const int per = (p.kb_total + p.splits - 1) / p.splits;
  t.split = split;
  t.kb0 = split * per;
  t.kb1 = min(p.kb_total, t.kb0 + per);
  return t;
}


// ------------------------------------------------------------------------------------------------------------------
// epilogues.  One thread = one accumulator row x (BN/2) columns, processed in 32-column chunks of the shared-memory
// accumulator tile (`t_addr`: word address of this thread's row at the half tile's first column).
// ------------------------------------------------------------------------------------------------------------------
constexpr float kLog2e = 1.4426950408889634f;
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ void load8(const float* p, float* o) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}
__device__ __forceinline__ void store8_bf16(bf16* dp, const float* o) {
  uint4 q;
  q.x = pack_bf16x2(o[0], o[1]); q.y = pack_bf16x2(o[2], o[3]);
  q.z = pack_bf16x2(o[4], o[5]); q.w = pack_bf16x2(o[6], o[7]);
  *reinterpret_cast<uint4*>(dp) = q;
}
__device__ __forceinline__ void load8_bf16(const bf16* sp, float* o) {
  const uint4 rr = *reinterpret_cast<const uint4*>(sp);
  const float2 r0 = unpack_bf16x2(rr.x), r1 = unpack_bf16x2(rr.y), r2 = unpack_bf16x2(rr.z), r3 = unpack_bf16x2(rr.w);
  o[0] = r0.x; o[1] = r0.y; o[2] = r1.x; o[3] = r1.y; o[4] = r2.x; o[5] = r2.y; o[6] = r3.x; o[7] = r3.y;
}

// Coalesced epilogue I/O.  A thread owns one accumulator ROW, so touching global memory directly would make every
// warp-level access hit 32 different rows with 16 bytes each (partial sectors -> L2 read-modify-write and DRAM reads
// on a pure write).  Each epilogue warp therefore owns a 4 KiB
// smem buffer holding a [32 rows][128 B] block (16-byte slots XOR-swizzled by row: conflict-free both ways); global
// traffic is 8 instructions of 4 rows x 128 contiguous bytes = whole cache lines, for outputs AND for the
// residual / ReLU-mask operands.
constexpr uint32_t STG_BYTES = 32 * 128;  // per epilogue warp

__device__ __forceinline__ uint32_t stg_addr(uint32_t stg, int row, int slot) {
  return stg + row * 128 + (((slot ^ row) & 7) << 4);
}
__device__ __forceinline__ void st_shared_v4u(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4u(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr)
               : "memory");
  return v;
}
// this lane's row: 32 bf16 values -> slots [4h, 4h+4)
__device__ __forceinline__ void stage_put_bf16(uint32_t stg, int lane, int h, const float* o) {
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const float* v = o + g * 8;
    st_shared_v4u(stg_addr(stg, lane, h * 4 + g), pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]),
                  pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
  }
}
__device__ __forceinline__ void stage_get_bf16(uint32_t stg, int lane, int h, float* o) {
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const uint4 q = ld_shared_v4u(stg_addr(stg, lane, h * 4 + g));
    const float2 a = unpack_bf16x2(q.x), b = unpack_bf16x2(q.y), c = unpack_bf16x2(q.z), d = unpack_bf16x2(q.w);
    float* v = o + g * 8;
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
  }
}
// this lane's row: 32 fp32 values -> all 8 slots
__device__ __forceinline__ void stage_put_f32(uint32_t stg, int lane, const float* o) {
#pragma unroll
  for (int g = 0; g < 8; ++g)
    st_shared_v4u(stg_addr(stg, lane, g), __float_as_uint(o[g * 4]), __float_as_uint(o[g * 4 + 1]),
                  __float_as_uint(o[g * 4 + 2]), __float_as_uint(o[g * 4 + 3]));
}
// smem block -> global rows [row0, row0+32) x 128 bytes starting at element column col0 (ESZ bytes per element)
// STREAM: st.global.cs (evict-first) for outputs that are far larger than L2 and would only push the operands out.
__device__ __forceinline__ void st_global_v4(void* p, const uint4& v, bool stream) {
  if (stream)
    asm volatile("st.global.cs.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
  else
    *reinterpret_cast<uint4*>(p) = v;
}
template <int ESZ, bool STREAM = false>
__device__ __forceinline__ void stage_flush(uint32_t stg, void* D, long long ldd, int row0, int col0, int M, int N,
                                            int lane) {
  constexpr int EPS = 16 / ESZ;  // elements per 16-byte slot
  __syncwarp();
  const int slot = lane & 7, rsub = lane >> 3;
  char* dst = reinterpret_cast<char*>(D) + ((long long)(row0 + rsub) * ldd + col0 + slot * EPS) * ESZ;
  const long long step = ldd * (4 * ESZ);
  // (slot ^ r) & 7 with r = 4 i + rsub: the low two bits of r are rsub's, bit 2 alternates with i
  const uint32_t a0 = stg + rsub * 128 + (((slot ^ rsub) & 7) << 4);
  const uint32_t a1 = stg + (rsub + 4) * 128 + (((slot ^ (rsub + 4)) & 7) << 4);
  if (row0 + 32 <= M && col0 + 8 * EPS <= N) {  // interior block (warp-uniform): no per-row guards
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint4 v = ld_shared_v4u(((i & 1) ? a1 : a0) + (i >> 1) * 1024);
      st_global_v4(dst, v, STREAM);
      dst += step;
    }
  } else {
    const bool col_ok = col0 + slot * EPS + EPS <= N;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint4 v = ld_shared_v4u(((i & 1) ? a1 : a0) + (i >> 1) * 1024);
      if (col_ok && row0 + i * 4 + rsub < M) st_global_v4(dst, v, STREAM);
      dst += step;
    }
  }
  __syncwarp();
}
// global bf16 rows -> smem block (zero where out of range)
__device__ __forceinline__ void stage_fetch_bf16(uint32_t stg, const bf16* src, long long ld, int row0, int col0, int M,
                                                 int N, int lane) {
  const int slot = lane & 7, rsub = lane >> 3;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = i * 4 + rsub;
    const int row = row0 + r, col = col0 + slot * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row < M && col + 8 <= N) v = __ldg(reinterpret_cast<const uint4*>(src + (long long)row * ld + col));
    st_shared_v4u(stg_addr(stg, r, slot), v.x, v.y, v.z, v.w);
  }
  __syncwarp();
}

// cp.async (L2 -> smem without registers), 16 bytes, zero-filled when `ok` is false
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, bool ok) {
  const uint32_t sz = ok ? 16u : 0u;  // src-size 0: nothing is read, the 16 bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// column sums of the staged [32 rows][64 bf16] block (the values exactly as they are written to D), stored into
// colsum[col0 .. col0+64) of this row block's workspace row: lane l owns columns 2l, 2l+1.  Rows >= M hold zeros (their
// `o` was zeroed).  The host adds the row blocks in order afterwards.
__device__ __forceinline__ void stage_colsum_bf16(uint32_t stg, float* colsum, int col0, int N, int lane) {
  __syncwarp();
  // word `lane` of row r sits at r*128 + (((lane>>2) ^ r) & 7)*16 + (lane&3)*4: the swizzle depends on r & 7 only, so 8
  // bases cover all 32 rows with immediate offsets (no address arithmetic inside the loop)
  const uint32_t w0 = stg + (lane & 3) * 4;
  const int slot = lane >> 2;
  uint32_t base[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) base[t] = w0 + t * 128 + (((slot ^ t) & 7) << 4);
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;  // two accumulator pairs: shorter dependency chains
#pragma unroll
  for (int q = 0; q < 4; ++q) {
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      uint32_t w;
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(base[t] + q * 1024) : "memory");
      const float2 f = unpack_bf16x2(w);
      if (t & 1) { s2 += f.x; s3 += f.y; } else { s0 += f.x; s1 += f.y; }
    }
  }
  const int col = col0 + 2 * lane;
  if (col < N) colsum[col] = s0 + s2;
  if (col + 1 < N) colsum[col + 1] = s1 + s3;
}

template <int CH>
__device__ __forceinline__ void epi_store(const GemmParams& p, uint32_t t_addr, int row, bool row_ok, int cbase,
                                          uint32_t stg, int row0, int lane) {
  static_assert(CH % 2 == 0, "epilogue works on pairs of 32-column chunks");
#pragma unroll 1
  for (int pc = 0; pc < CH / 2; ++pc) {
    const int colp = cbase + pc * 64;
    if (colp >= p.N) break;  // warp-uniform
    uint32_t rr2[2][32];
    acc_ld_x32(t_addr + (pc * 2) * 32, rr2[0]);
    acc_ld_x32(t_addr + (pc * 2 + 1) * 32, rr2[1]);
    if (p.residual) stage_fetch_bf16(stg, p.residual, p.ldr, row0, colp, p.M, p.N, lane);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int col0 = colp + h * 32;
      float o[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) o[j] = __uint_as_float(rr2[h][j]) * p.alpha;
      if (p.bias && col0 + 32 <= p.N) {
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          float b[8];
          load8(p.bias + col0 + g * 8, b);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[g * 8 + j] += b[j];
        }
      } else if (p.bias) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (col0 + j < p.N) o[j] += __ldg(p.bias + col0 + j);
      }
      if (p.relu) {
#pragma unroll
        for (int j = 0; j < 32; ++j) o[j] = fmaxf(o[j], 0.f);
      }
      if (p.residual) {
        float rr[32];
        stage_get_bf16(stg, lane, h, rr);
#pragma unroll
        for (int j = 0; j < 32; ++j) o[j] += rr[j];
      }
      if (p.out_f32) {  // 32 fp32 columns are a whole 128-byte line: flush per chunk
        if (p.residual) __syncwarp();
        // (fp32 output with a residual shares the buffer: the residual of chunk h was consumed above)
        if (p.residual && h == 0) {  // keep chunk 1's residual: spill it to registers before overwriting
          float keep[32];
          stage_get_bf16(stg, lane, 1, keep);
          stage_put_f32(stg, lane, o);
          stage_flush<4>(stg, p.D, p.ldd, row0, col0, p.M, p.N, lane);
          stage_put_bf16(stg, lane, 1, keep);
          __syncwarp();
        } else {
          stage_put_f32(stg, lane, o);
          stage_flush<4>(stg, p.D, p.ldd, row0, col0, p.M, p.N, lane);
        }
      } else {
        stage_put_bf16(stg, lane, h, o);
      }
    }
    if (!p.out_f32) stage_flush<2>(stg, p.D, p.ldd, row0, colp, p.M, p.N, lane);
  }
  (void)row; (void)row_ok;
}

// split_k == 1: D += alpha * acc with red.add (one contribution per element and call).  split_k > 1: D is this split's
// slice of a workspace and is overwritten; the host then adds the slices in split order (same result every run).
template <int CH>
__device__ __forceinline__ void epi_atomic(const GemmParams& p, float* D, int row, bool row_ok, int cbase,
                                           uint32_t t_addr) {
  const bool store = p.splits > 1;
#pragma unroll 1
  for (int c = 0; c < CH; ++c) {
    const int col0 = cbase + c * 32;
    if (col0 >= p.N) break;
    uint32_t r[32];
    acc_ld_x32(t_addr + c * 32, r);
    if (!row_ok) continue;
    float* dp = D + (long long)row * p.ldd + col0;
    if (store) {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (col0 + j < p.N) dp[j] = __uint_as_float(r[j]) * p.alpha;
    } else if (col0 + 32 <= p.N && (p.ldd & 3) == 0) {
#pragma unroll
      for (int j = 0; j < 32; j += 4)  // REDG.E.ADD.F32x4: one vector reduction per 16 bytes
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dp + j),
                     "f"(__uint_as_float(r[j]) * p.alpha), "f"(__uint_as_float(r[j + 1]) * p.alpha),
                     "f"(__uint_as_float(r[j + 2]) * p.alpha), "f"(__uint_as_float(r[j + 3]) * p.alpha)
                     : "memory");
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (col0 + j < p.N) atomicAdd(dp + j, __uint_as_float(r[j]) * p.alpha);
    }
  }
}

template <int CH>
__device__ __forceinline__ void epi_relu_bwd(const GemmParams& p, uint32_t t_addr, int row, bool row_ok, int cbase,
                                             uint32_t stg, int row0, int lane) {
#pragma unroll 1
  for (int pc = 0; pc < CH / 2; ++pc) {
    const int colp = cbase + pc * 64;
    if (colp >= p.N) break;
    uint32_t rr2[2][32];
    acc_ld_x32(t_addr + (pc * 2) * 32, rr2[0]);
    acc_ld_x32(t_addr + (pc * 2 + 1) * 32, rr2[1]);
    stage_fetch_bf16(stg, p.aux, p.ldaux, row0, colp, p.M, p.N, lane);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float am[32], o[32];
      stage_get_bf16(stg, lane, h, am);
#pragma unroll
      for (int j = 0; j < 32; ++j) o[j] = am[j] > 0.f ? __uint_as_float(rr2[h][j]) * p.alpha : 0.f;
      stage_put_bf16(stg, lane, h, o);  // in place: this lane overwrites the slots it just read
    }
    if (p.colsum) stage_colsum_bf16(stg, p.colsum + (long long)(row0 >> 5) * p.N, colp, p.N, lane);
    stage_flush<2>(stg, p.D, p.ldd, row0, colp, p.M, p.N, lane);
  }
  (void)row; (void)row_ok;
}

// per (row, half-tile): running max and sum exp of (acc + bias) over the valid vocabulary columns; label logit
template <int CH>
__device__ __forceinline__ void epi_ce_stats(const GemmParams& p, uint32_t t_addr, int row, bool row_ok, int cbase,
                                             int part_idx) {
  float run_max = -INFINITY, run_sum = 0.f;
  const int label = row_ok ? p.labels[row] : -1;
#pragma unroll 1
  for (int c = 0; c < CH; ++c) {
    const int col0 = cbase + c * 32;
    if (col0 >= p.N) break;
    uint32_t r[32];
    acc_ld_x32(t_addr + c * 32, r);
    if (!row_ok || col0 >= p.n_valid) continue;
    float v[32];
    if (col0 + 32 <= p.n_valid) {  // interior chunk (warp-uniform): no per-element masking
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        float b[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (p.bias) load8(p.bias + col0 + g * 8, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[g * 8 + j] = __uint_as_float(r[g * 8 + j]) + b[j];
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int col = col0 + j;
        v[j] = col < p.n_valid ? __uint_as_float(r[j]) + (p.bias ? __ldg(p.bias + col) : 0.f) : -INFINITY;
      }
    }
    if (label >= col0 && label < col0 + 32) {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (col0 + j == label) p.label_logit[row] = v[j];
    }
    float cmax = v[0];
#pragma unroll
    for (int j = 1; j < 32; ++j) cmax = fmaxf(cmax, v[j]);
    const float new_max = fmaxf(run_max, cmax);  // finite: at least one valid column in this chunk
    const float m2 = new_max * kLog2e;
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < 32; j += 2) {
      s0 += fast_exp2(fmaf(v[j], kLog2e, -m2));
      s1 += fast_exp2(fmaf(v[j + 1], kLog2e, -m2));
    }
    run_sum = run_sum * fast_exp2((run_max - new_max) * kLog2e) + (s0 + s1);
    run_max = new_max;
  }
  if (row_ok) {
    p.part_max[(long long)part_idx * p.M + row] = run_max;  // [n_parts][M]: a warp stores 32 consecutive floats
    p.part_sum[(long long)part_idx * p.M + row] = run_sum;
  }
}

// dlogits = alpha * (softmax - onehot), zero in the padded vocabulary columns.  alpha > 0 (checked by the host): it is
// folded into the exponent, alpha * 2^(x - l) = 2^(x - (l - log2 alpha)), which removes one multiply per element.
template <int CH>
__device__ __forceinline__ void epi_ce_grad(const GemmParams& p, uint32_t t_addr, int row, bool row_ok, int cbase,
                                            uint32_t stg, int row0, int lane) {
  const int label = row_ok ? p.labels[row] : -1;
  const float l2 = row_ok ? fmaf(p.lse[row], kLog2e, -log2f(p.alpha)) : 0.f;
#pragma unroll 1
  for (int pc = 0; pc < CH / 2; ++pc) {
    const int colp = cbase + pc * 64;
    if (colp >= p.N) break;
    uint32_t rr2[2][32];
    acc_ld_x32(t_addr + (pc * 2) * 32, rr2[0]);
    acc_ld_x32(t_addr + (pc * 2 + 1) * 32, rr2[1]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int col0 = colp + h * 32;
      const uint32_t* r = rr2[h];
      float o[32];
      if (col0 + 32 <= p.n_valid) {  // interior chunk (warp-uniform)
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          float b[8] = {0, 0, 0, 0, 0, 0, 0, 0};
          if (p.bias) load8(p.bias + col0 + g * 8, b);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            o[g * 8 + j] = fast_exp2(fmaf(__uint_as_float(r[g * 8 + j]) + b[j], kLog2e, -l2));
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int cc = col0 + j;
          o[j] = cc < p.n_valid
                     ? fast_exp2(fmaf(__uint_as_float(r[j]) + (p.bias ? __ldg(p.bias + cc) : 0.f), kLog2e, -l2))
                     : 0.f;
        }
      }
      if (label >= col0 && label < col0 + 32) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (col0 + j == label) o[j] -= p.alpha;
      }
      if (!row_ok) {  // rows past M: zeros (they are not stored, but the fused column sums read the staged block)
#pragma unroll
        for (int j = 0; j < 32; ++j) o[j] = 0.f;
      }
      stage_put_bf16(stg, lane, h, o);
    }
    if (p.colsum) stage_colsum_bf16(stg, p.colsum + (long long)(row0 >> 5) * p.N, colp, p.N, lane);
    stage_flush<2, true>(stg, p.D, p.ldd, row0, colp, p.M, p.N, lane);  // 4 GB of dlogits: stream past L2
  }
}

}  // namespace db200
