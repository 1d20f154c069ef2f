// GEMM kernel parameters, tile decoding and the epilogue routines that turn the shared-memory accumulator tile
// (wgmma.cuh: acc_store_smem / acc_ld_x32) of gemm_tc_kernel, or the accumulator fragments of gemm_pp_kernel, into
// global-memory results; the convolutions reuse the staging helpers.
#pragma once
#include "common.cuh"
#include "philox.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace db200 {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int GEMM_THREADS = 512;  // 4 control warps + 2 MMA warpgroups + 1 epilogue warpgroup
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
  db200_dropout drop;  // STORE with dropout (kernel instantiated with DROP = true): elementwise mask over [M][N]
  db200_ce_weights cew;  // weighted CE_GRAD (kernel instantiated with WCE = true): per-row class coefficients and z
  bf16* zout;            // GELU store: pre-activation z [M][ldz] (bf16), or NULL (inference: only h is written)
  long long ldz;
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

// o[j] *= keep ? scale : 0 for columns col0 .. col0 + 31 of row `row` (elementwise mask over [M][N]; col0 and N are
// multiples of 4, so the 32 columns are 8 whole Philox blocks)
__device__ __forceinline__ void dropout_row32(const db200_dropout& dr, int row, int N, int col0, float* o) {
  const uint64_t n0 = dropout_elem_block(dr, row, N, col0);
#pragma unroll
  for (int g = 0; g < 8; ++g) {
    const uint4 r = dropout_block(dr, n0 + g);
    o[4 * g + 0] *= dropout_mul(dr, r.x);
    o[4 * g + 1] *= dropout_mul(dr, r.y);
    o[4 * g + 2] *= dropout_mul(dr, r.z);
    o[4 * g + 3] *= dropout_mul(dr, r.w);
  }
}

template <int CH, bool DROP = false>
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
      if constexpr (DROP) dropout_row32(p.drop, row, p.N, col0, o);
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

// mtf's tanh GELU: gelu(x) = 0.5 x (1 + tanh(u)) = x s with s = sigma(2u) = 1 / (1 + 2^(-2 log2(e) u)) and
// u = sqrt(2/pi) (x + 0.044715 x^3).  ex2.approx and rcp.approx keep s within a few fp32 ulps *relative* over the whole
// range (tanh.approx's absolute error of ~2^-11 would be a large relative error in the negative tail); an exponent
// argument t carries a relative error of ~|t| ln2 2^-24 into s.  Where 1 + 2^t overflows or rcp underflows (z below
// about -10.1, where |gelu| < 2^-126 |z|), s is 0 and h is (-)0.  Large |x| overflows x^3 to +-inf, which gives s = 1
// or 0 exactly: finite z always yields a finite h.  +inf -> +inf; -inf and NaN -> NaN.
constexpr float kGeluA = 0.044715f;
constexpr float kGeluC2 = 1.5957691216057308f;    // 2 sqrt(2/pi)
constexpr float kGeluT = -2.3022082088626627f;    // -2 log2(e) sqrt(2/pi)
__device__ __forceinline__ float fast_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_s(float x) {
  return fast_rcp(1.f + fast_exp2(kGeluT * fmaf(kGeluA * x, x * x, x)));
}
// gelu'(x) = s + x s (1 - s) 2 sqrt(2/pi) (1 + 3 * 0.044715 x^2).  Where s is exactly 0 or 1, s (1 - s) = 0 and the
// result is exactly s (no 0 * inf from the overflowing x^2 term); 0 * x turns +-inf into NaN, as torch's float64 does.
__device__ __forceinline__ float gelu_grad(float x) {
  const float s = gelu_s(x);
  const float q = s * (1.f - s);
  return q == 0.f ? fmaf(0.f, x, s) : fmaf(x * q, kGeluC2 * fmaf(3.f * kGeluA, x * x, 1.f), s);
}

// GELU forward store: z = bf16(alpha acc + bias) is staged (and written to zout when it is given), read back as the
// rounded value and replaced in place by h = bf16(gelu(z)) evaluated in fp32, which goes to D.
template <int CH>
__device__ __forceinline__ void epi_gelu_store(const GemmParams& p, uint32_t t_addr, int cbase, uint32_t stg, int row0,
                                               int lane) {
#pragma unroll 1
  for (int pc = 0; pc < CH / 2; ++pc) {
    const int colp = cbase + pc * 64;
    if (colp >= p.N) break;  // warp-uniform
    uint32_t rr2[2][32];
    acc_ld_x32(t_addr + (pc * 2) * 32, rr2[0]);
    acc_ld_x32(t_addr + (pc * 2 + 1) * 32, rr2[1]);
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
      stage_put_bf16(stg, lane, h, o);
    }
    if (p.zout) stage_flush<2>(stg, p.zout, p.ldz, row0, colp, p.M, p.N, lane);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float z[32];
      stage_get_bf16(stg, lane, h, z);  // this lane's own row: no exchange between lanes
#pragma unroll
      for (int j = 0; j < 32; ++j) z[j] *= gelu_s(z[j]);
      stage_put_bf16(stg, lane, h, z);
    }
    stage_flush<2>(stg, p.D, p.ldd, row0, colp, p.M, p.N, lane);
  }
}

// GELU backward (dgrad of the MLP's first product): dZ = bf16(alpha acc * gelu'(z)), z read from aux; fused column
// sums as in RELU_BWD.  Rows and columns past the matrix read z = 0 and acc = 0, so they stage zeros.
template <int CH>
__device__ __forceinline__ void epi_gelu_bwd(const GemmParams& p, uint32_t t_addr, int cbase, uint32_t stg, int row0,
                                             int lane) {
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
      float o[32];
      stage_get_bf16(stg, lane, h, o);
#pragma unroll
      for (int j = 0; j < 32; ++j) o[j] = __uint_as_float(rr2[h][j]) * p.alpha * gelu_grad(o[j]);
      stage_put_bf16(stg, lane, h, o);  // in place: this lane overwrites the slots it just read
    }
    if (p.colsum) stage_colsum_bf16(stg, p.colsum + (long long)(row0 >> 5) * p.N, colp, p.N, lane);
    stage_flush<2>(stg, p.D, p.ldd, row0, colp, p.M, p.N, lane);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Gated MLP (GLU).  z = [zv | zg] is [M][2N] (value half first: DALLE-pytorch's chunk order), h = zv * act(zg) is
// [M][N].  The gate's nonlinearity a = bf16(act(zg)): GEGLU's zg s(zg) exactly as the GELU store evaluates it;
// ReGLU's zg > 0 ? zg : 0, which maps NaN (and -0) to +0 as the ReLU store's fmaxf does NaN.  h = bf16(zv a): the
// product of two bf16 values is exact in fp32 unless it leaves the normal range.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
template <bool GELU>
__device__ __forceinline__ float glu_act(float zg) {
  if constexpr (GELU) return round_bf16(zg * gelu_s(zg));
  else return zg > 0.f ? zg : 0.f;
}

// GLU forward store (the W1 product, N = the h width).  Tile n_blk holds value columns [64 n_blk, 64 n_blk + 64) in
// accumulator columns 0-63 and the matching gate columns N + 64 n_blk .. in 64-127 (the producer loads the two B
// slabs from there), so each thread has both halves of its row.  zv and zg = bf16(alpha acc + bias) go through the
// staging block (and to zout at their two offsets when it is given); zv stays in registers as the 32 packed words
// it was staged as while the block takes zg, then a and h = bf16(zv a) replace zg in place and h goes to D.
template <bool GELU>
__device__ __forceinline__ void epi_glu_store(const GemmParams& p, uint32_t t_addr, int colp, uint32_t stg, int row0,
                                              int lane) {
  uint32_t zv[32];  // columns 2 k, 2 k + 1 of this lane's value row
#pragma unroll
  for (int half = 0; half < 2; ++half) {  // 0: value, 1: gate
    const int zcol = half * p.N + colp;   // bias and z column of the half
    uint32_t rr2[2][32];
    acc_ld_x32(t_addr + half * 64, rr2[0]);
    acc_ld_x32(t_addr + half * 64 + 32, rr2[1]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float o[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) o[j] = __uint_as_float(rr2[h][j]) * p.alpha;
      if (p.bias) {  // N % 64 == 0: whole chunks
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          float b[8];
          load8(p.bias + zcol + h * 32 + g * 8, b);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[g * 8 + j] += b[j];
        }
      }
      stage_put_bf16(stg, lane, h, o);
    }
    if (p.zout) stage_flush<2>(stg, p.zout, p.ldz, row0, zcol, p.M, 2 * p.N, lane);
    if (half == 0) {
#pragma unroll
      for (int g = 0; g < 8; ++g) {  // this lane's own row: no exchange between lanes
        const uint4 q = ld_shared_v4u(stg_addr(stg, lane, g));
        zv[4 * g] = q.x; zv[4 * g + 1] = q.y; zv[4 * g + 2] = q.z; zv[4 * g + 3] = q.w;
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float o[32];
    stage_get_bf16(stg, lane, h, o);  // zg
#pragma unroll
    for (int j = 0; j < 32; j += 2) {
      const float2 v = unpack_bf16x2(zv[h * 16 + j / 2]);
      o[j] = v.x * glu_act<GELU>(o[j]);
      o[j + 1] = v.y * glu_act<GELU>(o[j + 1]);
    }
    stage_put_bf16(stg, lane, h, o);
  }
  stage_flush<2>(stg, p.D, p.ldd, row0, colp, p.M, p.N, lane);
}

// GLU backward (the dgrad dh = dbranch W2^T, N = the h width; D and aux are [M][2N]).  Half tile [colp, colp + 64) of
// dh = alpha acc (fp32, not rounded) reads zg, then zv, from the stored z and writes
//   dzv = bf16(dh a)                 a = bf16(act(zg)) as in the forward
//   dzg = bf16((dh act'(zg)) zv)     multiplied in this order; ReGLU's dh act'(zg) is zg > 0 ? dh : 0 (RELU_BWD's
//                                    mask convention), GEGLU's dh gelu'(zg)
// each through the staging block with its fused column sums (workspace rows of 2N columns).  Rows past M read z = 0
// and acc = 0, so they stage zeros.
template <bool GELU>
__device__ __forceinline__ void epi_glu_bwd(const GemmParams& p, uint32_t t_addr, int colp, uint32_t stg, int row0,
                                            int lane) {
  if (colp >= p.N) return;  // warp-uniform
  const int N2 = 2 * p.N;
  float dh[2][32];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    uint32_t r[32];
    acc_ld_x32(t_addr + h * 32, r);
#pragma unroll
    for (int j = 0; j < 32; ++j) dh[h][j] = __uint_as_float(r[j]) * p.alpha;
  }
  stage_fetch_bf16(stg, p.aux, p.ldaux, row0, p.N + colp, p.M, N2, lane);  // zg
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float o[32];
    stage_get_bf16(stg, lane, h, o);
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const float zg = o[j];
      o[j] = dh[h][j] * glu_act<GELU>(zg);
      if constexpr (GELU) dh[h][j] *= gelu_grad(zg);
      else dh[h][j] = zg > 0.f ? dh[h][j] : 0.f;
    }
    stage_put_bf16(stg, lane, h, o);  // in place: this lane overwrites the slots it just read
  }
  if (p.colsum) stage_colsum_bf16(stg, p.colsum + (long long)(row0 >> 5) * N2, colp, N2, lane);
  stage_flush<2>(stg, p.D, p.ldd, row0, colp, p.M, N2, lane);
  stage_fetch_bf16(stg, p.aux, p.ldaux, row0, colp, p.M, N2, lane);  // zv
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float o[32];
    stage_get_bf16(stg, lane, h, o);
#pragma unroll
    for (int j = 0; j < 32; ++j) o[j] = dh[h][j] * o[j];
    stage_put_bf16(stg, lane, h, o);
  }
  if (p.colsum) stage_colsum_bf16(stg, p.colsum + (long long)(row0 >> 5) * N2, p.N + colp, N2, lane);
  stage_flush<2>(stg, p.D, p.ldd, row0, p.N + colp, p.M, N2, lane);
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

// Weighted CE_GRAD: dlogits = a (c' softmax - onehot) with a = a_text for rows t with t mod period < text_rows, else
// a_image, and c' = 1 + 2 z lse (the z-loss z lse^2 adds 2 z lse softmax to the gradient).  c = a c' is formed once per
// row; |c| is folded into the exponent as in epi_ce_grad and its sign applied afterwards.  c = 0 (a zero-weight class,
// or c' = 0) gives log2 |c| = -inf, hence exp2(-inf) = 0: the row's softmax term is exactly 0, as is its label term.
template <int CH>
__device__ __forceinline__ void epi_ce_grad_weighted(const GemmParams& p, uint32_t t_addr, int row, bool row_ok,
                                                     int cbase, uint32_t stg, int row0, int lane) {
  const int label = row_ok ? p.labels[row] : -1;
  float a = 0.f, l2 = 0.f;
  bool neg = false;
  if (row_ok) {
    a = (row % p.cew.period) < p.cew.text_rows ? p.cew.a_text : p.cew.a_image;
    const float lse = p.lse[row];
    const float c = a * fmaf(2.f * p.cew.z_loss, lse, 1.f);
    neg = c < 0.f;
    l2 = fmaf(lse, kLog2e, -log2f(fabsf(c)));
  }
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
      if (neg) {  // only rows with lse < -1 / (2 z)
#pragma unroll
        for (int j = 0; j < 32; ++j) o[j] = -o[j];
      }
      if (label >= col0 && label < col0 + 32) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (col0 + j == label) o[j] -= a;
      }
      if (!row_ok) {
#pragma unroll
        for (int j = 0; j < 32; ++j) o[j] = 0.f;
      }
      stage_put_bf16(stg, lane, h, o);
    }
    if (p.colsum) stage_colsum_bf16(stg, p.colsum + (long long)(row0 >> 5) * p.N, colp, p.N, lane);
    stage_flush<2, true>(stg, p.D, p.ldd, row0, colp, p.M, p.N, lane);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// fragment epilogues (gemm_pp_kernel).  A warpgroup holds a whole 128 x 128 tile as two m64n128 accumulator fragments
// (wgmma.cuh): thread t keeps, for chain c, 8-column group i and row half h, the pair d[frag_idx(c, i, h) + {0, 1}] =
// tile row 64 c + 16 (t / 32) + 8 h + (t % 32) / 4, columns 8 i + 2 (t % 4) + {0, 1}.  The elementwise math runs on
// those registers in place, with the per-element expressions of the row-per-thread epilogues above, so both kernels
// round identically.  Global traffic keeps the staging discipline: rows [32 b, 32 b + 32) of the tile live in the
// two warps 2 (b % 2), 2 (b % 2) + 1 of chain b / 2, which fill that row block's [32 rows][128 B] staging block
// together (a 64-thread named barrier around it); one of the two then runs the unchanged stage_fetch_bf16 /
// stage_colsum_bf16 / stage_flush on it.  A warp pair serves two blocks (one per chain) and each warp owns one.
// gemm_wide_kernel's warpgroups hold a 64 x 256 slice as one m64n256 fragment, whose two halves are the m64n128
// fragments of columns [0, 128) and [128, 256): the same registers with the chains side by side instead of stacked.
// Template parameter CW says which: 0 (chain c at rows 64 c) or 128 (chain c at columns 128 c); warp pair b / 2 of a
// wide warpgroup then stages rows [32 b, 32 b + 32) of its slice for both column halves.
// ------------------------------------------------------------------------------------------------------------------
__host__ __device__ constexpr int frag_idx(int c, int i, int h) { return c * 64 + 4 * i + 2 * h; }

struct FragCtx {
  uint32_t own_stg;  // the staging block this warp fetches, sums and flushes (its pair's block of chain `own`)
  uint32_t a[2];    // this thread's 4-byte word in row half 0 of each block at column group 0 (swizzle folded in)
  int lane, q;      // q = lane % 4: the thread's column pair inside every 8-column group
  int row;          // tile row of (chain 0, half 0): 16 (t / 32) + (t % 32) / 4
  int own_row0;     // first tile row of that block
  int own_col;      // its first column, relative to the chain 0 column of the same 64-column group
  int bar;          // named barrier of the warp pair
};
template <int CW>
__device__ __forceinline__ FragCtx frag_ctx(uint32_t stg_wg, int wg_thread, int bar0) {
  static_assert(CW == 0 || CW == 128, "chains stacked in rows or side by side in columns");
  FragCtx f;
  const int w = wg_thread >> 5;
  f.lane = wg_thread & 31;
  f.q = f.lane & 3;
  f.row = 16 * w + (f.lane >> 2);
  f.own_row0 = (CW ? 0 : 64 * (w & 1)) + 32 * (w >> 1);
  f.own_col = CW * (w & 1);
  f.own_stg = stg_wg + (2 * (w & 1) + (w >> 1)) * STG_BYTES;
  f.bar = bar0 + (w >> 1);
  const int r = 16 * (w & 1) + (f.lane >> 2);  // row inside the block; r % 8 == lane / 4 for both row halves
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    f.a[c] = stg_wg + (2 * c + (w >> 1)) * STG_BYTES + r * 128 + ((f.lane >> 2) << 4) + 4 * f.q;
  }
  return f;
}
__device__ __forceinline__ void pair_sync(const FragCtx& f) { named_bar_sync(f.bar, 64); }
// 16-byte slot `slot` of the thread's row (half h): the row's XOR swizzle is already in f.a, blocks are 128 B aligned
__device__ __forceinline__ uint32_t frag_addr(const FragCtx& f, int c, int h, int slot) {
  return (f.a[c] + h * 1024) ^ (slot << 4);
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
// columns [64 hp, 64 hp + 64) of the tile as bf16 into both blocks
__device__ __forceinline__ void frag_put_bf16(const FragCtx& f, const float (&d)[128], int hp) {
#pragma unroll
  for (int c = 0; c < 2; ++c)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int k = frag_idx(c, 8 * hp + i, h);
        st_shared_u32(frag_addr(f, c, h, i), pack_bf16x2(d[k], d[k + 1]));
      }
}
// columns [32 s, 32 s + 32) of the tile as fp32 into both blocks: column 8 i + 2 q is word 2 q of slots 2 i, 2 i + 1
__device__ __forceinline__ void frag_put_f32(const FragCtx& f, const float (&d)[128], int s) {
#pragma unroll
  for (int c = 0; c < 2; ++c)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int k = frag_idx(c, 4 * s + i, h);
        const uint32_t row_base = (f.a[c] + h * 1024 - 4 * f.q) ^ ((2 * i + (f.q >> 1)) << 4);
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(row_base + 8 * (f.q & 1)), "f"(d[k]), "f"(d[k + 1])
                     : "memory");
      }
}
// bias of the thread's column pairs in columns [col0, col0 + 64), zero at and past `limit` (even or odd)
__device__ __forceinline__ void frag_bias(const float* bias, int col0, int q, int limit, float2 (&b)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int col = col0 + 8 * i + 2 * q;
    b[i] = make_float2(0.f, 0.f);
    if (!bias) continue;
    if (col + 1 < limit) b[i] = __ldg(reinterpret_cast<const float2*>(bias + col));
    else if (col < limit) b[i].x = __ldg(bias + col);
  }
}
// the owner's work on its staged bf16 block: fused column sums (when asked for) and the flush to D
template <bool STREAM>
__device__ __forceinline__ void frag_flush_bf16(const GemmParams& p, const FragCtx& f, int m0, int colp, bool colsum) {
  const int row0 = m0 + f.own_row0, col0 = colp + f.own_col;
  if (colsum) stage_colsum_bf16(f.own_stg, p.colsum + (long long)(row0 >> 5) * p.N, col0, p.N, f.lane);
  stage_flush<2, STREAM>(f.own_stg, p.D, p.ldd, row0, col0, p.M, p.N, f.lane);
}

// m0, n0: the fragment's first row and column (chain 0).  Side-by-side chains past N stage values the bounded
// fetches, sums and flushes then ignore.
template <int CW>
__device__ __forceinline__ void frag_store(const GemmParams& p, float (&d)[128], const FragCtx& f, int m0, int n0) {
#pragma unroll
  for (int hp = 0; hp < 2; ++hp) {
    const int colp = n0 + hp * 64;
    if (colp >= p.N) break;  // uniform over the tile
    if (p.residual) {
      stage_fetch_bf16(f.own_stg, p.residual, p.ldr, m0 + f.own_row0, colp + f.own_col, p.M, p.N, f.lane);
      pair_sync(f);
    }
    float2 b[CW ? 2 : 1][8];
#pragma unroll
    for (int c = 0; c < (CW ? 2 : 1); ++c) frag_bias(p.bias, colp + CW * c, f.q, p.N, b[c]);
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int k = frag_idx(c, 8 * hp + i, h);
          d[k] = d[k] * p.alpha;
          d[k + 1] = d[k + 1] * p.alpha;
        }
        if (p.bias) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int k = frag_idx(c, 8 * hp + i, h);
            d[k] += b[CW ? c : 0][i].x;
            d[k + 1] += b[CW ? c : 0][i].y;
          }
        }
        if (p.relu) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int k = frag_idx(c, 8 * hp + i, h);
            d[k] = fmaxf(d[k], 0.f);
            d[k + 1] = fmaxf(d[k + 1], 0.f);
          }
        }
        if (p.residual) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int k = frag_idx(c, 8 * hp + i, h);
            const float2 r = unpack_bf16x2(ld_shared_u32(frag_addr(f, c, h, i)));
            d[k] += r.x;
            d[k + 1] += r.y;
          }
        }
      }
    if (!p.out_f32) {  // in place: every thread overwrites the residual words it has just read
      frag_put_bf16(f, d, hp);
      pair_sync(f);
      frag_flush_bf16<false>(p, f, m0, colp, false);
      pair_sync(f);
    } else {
      if (p.residual) pair_sync(f);  // fp32 words land on other threads' residual words
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        frag_put_f32(f, d, 2 * hp + s);
        pair_sync(f);
        stage_flush<4>(f.own_stg, p.D, p.ldd, m0 + f.own_row0, colp + f.own_col + 32 * s, p.M, p.N, f.lane);
        pair_sync(f);
      }
    }
  }
}

template <int CW>
__device__ __forceinline__ void frag_relu_bwd(const GemmParams& p, float (&d)[128], const FragCtx& f, int m0, int n0) {
#pragma unroll
  for (int hp = 0; hp < 2; ++hp) {
    const int colp = n0 + hp * 64;
    if (colp >= p.N) break;
    stage_fetch_bf16(f.own_stg, p.aux, p.ldaux, m0 + f.own_row0, colp + f.own_col, p.M, p.N, f.lane);
    pair_sync(f);
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int k = frag_idx(c, 8 * hp + i, h);
          const uint32_t addr = frag_addr(f, c, h, i);
          const float2 am = unpack_bf16x2(ld_shared_u32(addr));
          const float o0 = am.x > 0.f ? d[k] * p.alpha : 0.f;
          const float o1 = am.y > 0.f ? d[k + 1] * p.alpha : 0.f;
          st_shared_u32(addr, pack_bf16x2(o0, o1));  // in place: the word this thread has just read
        }
    pair_sync(f);
    frag_flush_bf16<false>(p, f, m0, colp, p.colsum != nullptr);
    pair_sync(f);
  }
}

__device__ __forceinline__ void frag_ce_grad(const GemmParams& p, float (&d)[128], const FragCtx& f, int m0, int n0) {
  int label[2][2];
  float l2[2][2];
  bool row_ok[2][2];
#pragma unroll
  for (int c = 0; c < 2; ++c)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m0 + 64 * c + 8 * h + f.row;
      row_ok[c][h] = row < p.M;
      label[c][h] = row_ok[c][h] ? p.labels[row] : -1;
      l2[c][h] = row_ok[c][h] ? fmaf(p.lse[row], kLog2e, -log2f(p.alpha)) : 0.f;
    }
#pragma unroll
  for (int hp = 0; hp < 2; ++hp) {
    const int colp = n0 + hp * 64;
    if (colp >= p.N) break;
    float2 b[8];
    frag_bias(p.bias, colp, f.q, p.n_valid, b);
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int k = frag_idx(c, 8 * hp + i, h);
          const int col = colp + 8 * i + 2 * f.q;
          float o0 = col < p.n_valid ? fast_exp2(fmaf(d[k] + b[i].x, kLog2e, -l2[c][h])) : 0.f;
          float o1 = col + 1 < p.n_valid ? fast_exp2(fmaf(d[k + 1] + b[i].y, kLog2e, -l2[c][h])) : 0.f;
          if (col == label[c][h]) o0 -= p.alpha;
          if (col + 1 == label[c][h]) o1 -= p.alpha;
          // rows past M: zeros (they are not stored, but the fused column sums read the staged block)
          d[k] = row_ok[c][h] ? o0 : 0.f;
          d[k + 1] = row_ok[c][h] ? o1 : 0.f;
        }
    frag_put_bf16(f, d, hp);
    pair_sync(f);
    frag_flush_bf16<true>(p, f, m0, colp, p.colsum != nullptr);  // 4 GB of dlogits: stream past L2
    pair_sync(f);
  }
}

}  // namespace db200
