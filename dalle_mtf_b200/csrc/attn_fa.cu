// K4 — causal flash attention on wgmma (sm_90a): forward, and the backward as two kernels (dQ per query block, dK / dV
// per key block), so that no gradient needs atomics.
//
// One CTA = one warpgroup = 64 rows of one (batch, head).  Tiles of 64 rows x dh are brought into shared memory with
// cp.async in the 128B-swizzled layout of the wgmma descriptors ([dh / 64 atoms][64 rows][64 bf16]); the same K / V /
// Q / dO tile serves as a K-major operand (rows = the contracted dimension's partner) and, read through an MN-major
// descriptor, as the B operand of the products that contract over its rows.  Logits, softmax and gradients stay in the
// fp32 accumulator fragments; P and dS are packed to bf16 in registers and fed to the next wgmma as its A operand.
//
// Layout: qkv bf16 [B][S][3][H][dh], out / dout bf16 [B][S][H][dh], lse / delta f32 [B][H][S], dqkv like qkv.
//
// LOCAL (sliding-window attention, mtf local_attention_1d with fully_autoregressive=True, src/dalle_mtf/models.py:
// 257-273): query i sees key j iff i - radius < j <= i.  The loops visit only the key (query) blocks that intersect that
// band and the masks add the lower edge; the global (causal) instantiations compile without either.
//
// AXIAL (DALL-E's row and column attention, DALLE-pytorch's "axial_row" / "axial_col"): text length TL, image grid
// W x W, position p >= TL is image token k = p - TL at row k / W, column k % W.  Text queries are causal; an image
// query sees every text key and the image keys of its own row (column) at or before it.  The kernels walk the rows in
// "kernel order" t: t = p for a row layer and for text rows; the image rows of a column layer are taken column-major,
// u = t - TL, p = TL + (u % W) W + u / W.  In kernel order both layers are one mask: t_k <= t_q and (t_k < TL or
// t_k >= the start TL + ((t_q - TL) / W) W of t_q's segment), i.e. a text prefix plus causal attention inside
// segments of W rows.  Every global access (tile loads, stores, lse / delta) goes through the row map, so the tensor
// layouts are those of the other instantiations; rows whose p >= S (a shorter prefill) are absent: zero-filled,
// never stored, and a present query never sees one.
//
// CONV (DALL-E's convolutional attention, DALLE-pytorch's SparseConvCausalAttention at dilation 1): the grid of AXIAL,
// kernel size k.  Text queries are causal; the image query at (r, c) sees every text key and the image keys (r', c')
// with r - k < r' <= r and c - k < c' <= c, the k x k window above and to the left of it.  Rows stay in raster order
// (no row map).  Every visible key precedes its query, but the mask is not a band: (r - 1, c + 1) is earlier and
// outside the window.  The loops visit the text blocks and the band of blocks from the window's top row to the
// query; each tile's mask tests the window from grid coordinates stepped along the thread's columns.
//
// SPARSE (DeepSpeed-style block-sparse attention, DALLE-pytorch's SparseAttention): a per-layer table of 16-bit tile
// masks, mask[qt * pitch + kt] for the 64 x 64 tile of query block qt and key block kt <= qt.  Bit 4 a + c set: the 16
// queries 64 qt + 16 a .. + 15 see the 16 keys 64 kt + 16 c .. + 15, under the causal mask (key <= query, key < S).
// The forward and dQ kernels visit, in ascending order, the key blocks whose mask is non-zero; the dK / dV kernel the
// query blocks.  Warp w of the warpgroup holds the fragment rows 16 w .. 16 w + 15 and element i of a row lies in
// column block i / 2, so each thread tests one nibble of the mask.  The table's pitch is independent of S, so that a
// prefill shorter than the table reads the rows it covers.
#include "gemm_common.cuh"  // cp.async helpers
#include "philox.cuh"
#include "wgmma.cuh"

namespace db200 {
namespace {

constexpr int FA_ROWS = 64;
constexpr float kLn2 = 0.6931471805599453f;

// 64 rows x DH bf16 (row r at src + r * ld, rows >= n_rows zero-filled) -> swizzled smem tile; the caller commits
template <int DH>
__device__ __forceinline__ void fa_load_tile(uint32_t dst, const bf16* src, long long ld, int n_rows) {
  constexpr int CPR = DH / 8;  // 16-byte chunks per row
#pragma unroll
  for (int i = 0; i < FA_ROWS * CPR / 128; ++i) {
    const int idx = threadIdx.x + 128 * i;
    const int r = idx / CPR, c = idx % CPR;
    const bool ok = r < n_rows;
    const uint32_t off = (c >> 3) * (FA_ROWS * 128) + r * 128 + ((((c & 7) ^ (r & 7)) & 7) << 4);
    cp_async16_zfill(dst + off, ok ? src + (long long)r * ld + c * 8 : src, ok);
  }
}
// all outstanding tile loads have landed and are visible to the wgmma (async) proxy of every thread
__device__ __forceinline__ void fa_tiles_ready() {
  cp_async_commit();
  cp_async_wait<0>();
  fence_proxy_async_smem();
  __syncthreads();
}

// K-major descriptor of k-step ks (16 columns) of a [64 rows][DH] tile: 64-column atoms 8 KiB apart
__device__ __forceinline__ uint64_t fa_kdesc(uint32_t tile, int ks) {
  return smem_desc_sw128(tile + (ks >> 2) * (FA_ROWS * 128) + (ks & 3) * 32, 0, 1024);
}
// MN-major descriptor of k-step ks (16 rows) of the same tile used as a B operand with N = DH
__device__ __forceinline__ uint64_t fa_ndesc(uint32_t tile, int ks) {
  return smem_desc_sw128(tile + ks * 2048, FA_ROWS * 128, 1024);
}

// S[64 x 64] = A_tile[64 x DH] * B_tile[64 x DH]^T (both K-major)
template <int DH>
__device__ __forceinline__ void fa_qk(float* s, uint32_t a_tile, uint32_t b_tile) {
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < DH / 16; ++ks) wgmma_m64n64<0, 0>(s, fa_kdesc(a_tile, ks), fa_kdesc(b_tile, ks), ks > 0);
  wgmma_commit();
  wgmma_wait<0>();
}
// acc[64 x DH] += P[64 x 64] (registers, fp32 fragment packed to bf16 here) * tile[64 x DH]
// DROP: fragment element x is multiplied by (bit x of kb) ? sc : 0 on the way (dropout of P)
template <int DH, bool DROP = false>
__device__ __forceinline__ void fa_pv(float* acc, const float* p, uint32_t tile, uint32_t kb = 0u, float sc = 1.f) {
  uint32_t a[4][4];
  auto pk = [&](int x) { return DROP ? (((kb >> x) & 1u) ? p[x] * sc : 0.f) : p[x]; };
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = pack_bf16x2(pk(8 * ks + 0), pk(8 * ks + 1));
    a[ks][1] = pack_bf16x2(pk(8 * ks + 2), pk(8 * ks + 3));
    a[ks][2] = pack_bf16x2(pk(8 * ks + 4), pk(8 * ks + 5));
    a[ks][3] = pack_bf16x2(pk(8 * ks + 6), pk(8 * ks + 7));
  }
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    if constexpr (DH == 64) wgmma_rs_m64n64<1>(acc, a[ks], fa_ndesc(tile, ks), 1u);
    else wgmma_rs_m64n128<1>(acc, a[ks], fa_ndesc(tile, ks), 1u);
  }
  wgmma_commit();
  wgmma_wait<0>();
}

// fragment coordinates: element (i, h, e) of an m64 x N accumulator sits at row fr + 8 h, column 8 i + fc + e
struct Frag {
  int fr, fc;
  __device__ __forceinline__ Frag() {
    const int t = threadIdx.x & 127, lane = t & 31;
    fr = 16 * (t >> 5) + (lane >> 2);
    fc = 2 * (lane & 3);
  }
};
// Keep bits of this thread's 32 fragment elements of a 64 x 64 attention-weight tile (bit x = element x) whose first
// row / column are r0 / c0.  QROWS: rows are queries and columns keys (forward, dQ); else rows are keys and columns
// queries (dK / dV).  The two columns fc, fc + 1 of a row share one 2 x 2 block, so each Philox call serves two elements.
template <bool QROWS>
__device__ __forceinline__ uint32_t fa_keep_bits(const db200_dropout& dr, int b, int h, int H, int S2, int r0, int c0,
                                                 const Frag& f) {
  uint32_t kb = 0u;
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = r0 + f.fr + 8 * hh, col = c0 + 8 * i + f.fc;  // col is even
      const uint4 r = dropout_block(dr, QROWS ? dropout_attn_block(dr, b, h, H, S2, row, col)
                                              : dropout_attn_block(dr, b, h, H, S2, col, row));
      // word of (query i, key j) = 2 (i & 1) + (j & 1)
      const uint32_t w0 = QROWS ? ((row & 1) ? r.z : r.x) : ((row & 1) ? r.y : r.x);
      const uint32_t w1 = QROWS ? ((row & 1) ? r.w : r.y) : ((row & 1) ? r.w : r.z);
      const int x = 4 * i + 2 * hh;
      kb |= (uint32_t)(w0 >= dr.threshold) << x;
      kb |= (uint32_t)(w1 >= dr.threshold) << (x + 1);
    }
  return kb;
}
__device__ __forceinline__ float fa_keep_mul(uint32_t kb, int x, float sc) { return ((kb >> x) & 1u) ? sc : 0.f; }

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// store an m64 x DH fp32 fragment (times `mul`) as bf16 rows r < n_rows of dst (row stride ld)
template <int DH>
__device__ __forceinline__ void fa_store_rows(bf16* dst, long long ld, const float* acc, const float (&mul)[2],
                                              int n_rows, const Frag& f) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = f.fr + 8 * h;
    if (r >= n_rows) continue;
    bf16* d = dst + (long long)r * ld + f.fc;
#pragma unroll
    for (int i = 0; i < DH / 8; ++i)
      *reinterpret_cast<uint32_t*>(d + 8 * i) = pack_bf16x2(acc[4 * i + 2 * h] * mul[h], acc[4 * i + 2 * h + 1] * mul[h]);
  }
}

template <int DH>
constexpr size_t fa_smem(int tiles) { return 1024 + size_t(tiles) * FA_ROWS * DH * 2 + 2 * FA_ROWS * 4; }

// ---- AXIAL: geometry and row map.  rows = kernel-order rows the grid covers (S for a row layer).
struct FaAxial {
  int text_len, grid_w, axis, rows;
};
// sequence position of kernel-order row t, or -1 when the row is absent
__device__ __forceinline__ int fa_axial_pos(const FaAxial& a, int S, int t) {
  if (t >= a.rows) return -1;
  int p = t;
  if (a.axis && t >= a.text_len) {
    const int u = t - a.text_len;
    p = a.text_len + (u % a.grid_w) * a.grid_w + u / a.grid_w;
  }
  return p < S ? p : -1;
}
// first kernel-order row of t's segment (0 for a text row: every key up to t)
__device__ __forceinline__ int fa_axial_seg_start(const FaAxial& a, int t) {
  return t < a.text_len ? 0 : a.text_len + (t - a.text_len) / a.grid_w * a.grid_w;
}
// fa_load_tile of kernel-order rows t0 .. t0 + 63: row t at base + p(t) * ld, absent rows zero-filled
template <int DH>
__device__ __forceinline__ void fa_load_tile_axial(uint32_t dst, const bf16* base, long long ld, const FaAxial& a,
                                                   int S, int t0) {
  constexpr int CPR = DH / 8;
#pragma unroll
  for (int i = 0; i < FA_ROWS * CPR / 128; ++i) {
    const int idx = threadIdx.x + 128 * i;
    const int r = idx / CPR, c = idx % CPR;
    const int p = fa_axial_pos(a, S, t0 + r);
    const bool ok = p >= 0;
    const uint32_t off = (c >> 3) * (FA_ROWS * 128) + r * 128 + ((((c & 7) ^ (r & 7)) & 7) << 4);
    cp_async16_zfill(dst + off, ok ? base + (long long)p * ld + c * 8 : base, ok);
  }
}
// fa_store_rows of kernel-order rows t0 .. t0 + 63 to base + p(t) * ld (present rows only)
template <int DH>
__device__ __forceinline__ void fa_store_rows_axial(bf16* base, long long ld, const float* acc, const float (&mul)[2],
                                                    const FaAxial& a, int S, int t0, const Frag& f) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int p = fa_axial_pos(a, S, t0 + f.fr + 8 * h);
    if (p < 0) continue;
    bf16* d = base + (long long)p * ld + f.fc;
#pragma unroll
    for (int i = 0; i < DH / 8; ++i)
      *reinterpret_cast<uint32_t*>(d + 8 * i) = pack_bf16x2(acc[4 * i + 2 * h] * mul[h], acc[4 * i + 2 * h + 1] * mul[h]);
  }
}
// key blocks of query block qb (forward, dQ): the text blocks [0, jt), then the blocks from js (the block of the segment
// start of the block's first image query) to qb.  No block is visited twice.
__device__ __forceinline__ void fa_axial_key_blocks(const FaAxial& a, int qb, int& jt, int& js) {
  jt = (a.text_len + FA_ROWS - 1) / FA_ROWS;
  const int t = max(qb * FA_ROWS, a.text_len);
  js = t < (qb + 1) * FA_ROWS ? fa_axial_seg_start(a, t) / FA_ROWS : jt;
}
__device__ __forceinline__ int fa_axial_next(int j, int jt, int js) { return (j + 1 >= jt && j + 1 < js) ? js : j + 1; }
// query blocks of key block kb (dK / dV): [kb, end).  A block holding a text key sees every later query; an image key
// block the queries up to the end of the last segment it touches.
__device__ __forceinline__ int fa_axial_query_end(const FaAxial& a, int kb) {
  const int nq = (a.rows + FA_ROWS - 1) / FA_ROWS, k0 = kb * FA_ROWS;
  if (k0 < a.text_len) return nq;
  const int last = min(k0 + FA_ROWS - 1, a.rows - 1);
  const int seg_end = fa_axial_seg_start(a, last) + a.grid_w - 1;
  return min(nq, seg_end / FA_ROWS + 1);
}

// ---- CONV: geometry (kernel >= 1).  Rows are sequence positions.
struct FaConv {
  int text_len, grid_w, kernel;
};
// grid row / column of position p, or row -1 for a text position
__device__ __forceinline__ void fa_conv_rc(const FaConv& c, int p, int& r, int& col) {
  const int u = p - c.text_len;
  r = u < 0 ? -1 : u / c.grid_w;
  col = u < 0 ? 0 : u - (u / c.grid_w) * c.grid_w;
}
// Visible bits of this thread's 32 fragment elements of a 64 x 64 tile (bit x = element x, as fa_keep_bits) whose first
// row / column are r0 / c0; rows and columns >= S are absent.  QROWS: rows are queries and columns keys (forward, dQ);
// else rows are keys and columns queries (dK / dV).  rr / rc: grid row / column of the thread's two rows (fa_conv_rc).
// The grid coordinates of the columns are stepped from one division per tile (floor division: a text column has a
// negative row, and stepping carries it into the image rows).
template <bool QROWS>
__device__ __forceinline__ uint32_t fa_conv_vis_bits(const FaConv& cv, int S, int r0, int c0, const int (&rr)[2],
                                                     const int (&rc)[2], const Frag& f) {
  const int u0 = c0 + f.fc - cv.text_len;
  int gr = u0 >= 0 ? u0 / cv.grid_w : -((cv.grid_w - 1 - u0) / cv.grid_w);
  int gc = u0 - gr * cv.grid_w;
  uint32_t bits = 0u;
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int col = c0 + 8 * i + f.fc + e;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = r0 + f.fr + 8 * hh;
        const bool vis =
            QROWS ? row < S && col <= row &&
                        (col < cv.text_len || (gr > rr[hh] - cv.kernel && gc <= rc[hh] && gc > rc[hh] - cv.kernel))
                  : col < S && row <= col &&
                        (row < cv.text_len || (gr - rr[hh] < cv.kernel && gc >= rc[hh] && gc - rc[hh] < cv.kernel));
        bits |= (uint32_t)vis << (4 * i + 2 * hh + e);
      }
      gc += e == 0 ? 1 : 7;  // the next column: col + 1, then col + 7 = the next i's first
      while (gc >= cv.grid_w) {
        gc -= cv.grid_w;
        ++gr;
      }
    }
  return bits;
}
// key blocks of query block qb (forward, dQ): the text blocks [0, jt), then the blocks from js (the block holding the
// first position of the window's top row, grid row max(0, r0 - k + 1), for the block's first image query at row r0) to
// qb.  With fa_axial_next no block is visited twice.
__device__ __forceinline__ void fa_conv_key_blocks(const FaConv& c, int qb, int& jt, int& js) {
  jt = (c.text_len + FA_ROWS - 1) / FA_ROWS;
  const int t = max(qb * FA_ROWS, c.text_len);
  const int top = max(0, (t - c.text_len) / c.grid_w - c.kernel + 1);
  js = t < (qb + 1) * FA_ROWS ? (c.text_len + top * c.grid_w) / FA_ROWS : jt;
}
// query blocks of key block kb (dK / dV): [kb, end).  A block holding a text key sees every later query; an image key
// is seen up to (k - 1) rows and k - 1 columns later, i.e. at most min(k - 1, W - 1) (W + 1) positions after it.
__device__ __forceinline__ int fa_conv_query_end(const FaConv& c, int S, int kb) {
  const int nq = (S + FA_ROWS - 1) / FA_ROWS, k0 = kb * FA_ROWS;
  if (k0 < c.text_len) return nq;
  const long long last = min(k0 + FA_ROWS - 1, S - 1);
  const long long reach = last + (long long)(min(c.kernel, c.grid_w) - 1) * (c.grid_w + 1);
  return (int)min((long long)nq, reach / FA_ROWS + 1);
}

// ---- SPARSE: tile-mask table (pitch >= the number of 64-row blocks of S)
struct FaSparse {
  const uint16_t* mask;
  int pitch;
};
__device__ __forceinline__ uint32_t fa_sparse_tile(const FaSparse& sp, int qt, int kt) {
  return sp.mask[(long long)qt * sp.pitch + kt];
}
// the first key block after j (<= qb) with a non-zero mask in query block qb's row, or qb + 1
__device__ __forceinline__ int fa_sparse_next_key(const FaSparse& sp, int qb, int j) {
  for (++j; j <= qb && fa_sparse_tile(sp, qb, j) == 0u; ++j) {
  }
  return j;
}
// the first query block after i (< nq) with a non-zero mask in key block kb's column, or nq
__device__ __forceinline__ int fa_sparse_next_query(const FaSparse& sp, int kb, int i, int nq) {
  for (++i; i < nq && fa_sparse_tile(sp, i, kb) == 0u; ++i) {
  }
  return i;
}
// Visible bits of this thread's 32 fragment elements (bit x = element x, as fa_conv_vis_bits) of the tile with mask tm
// whose first row / column are r0 / c0.  QROWS: rows are queries and columns keys (forward, dQ); else rows are keys
// and columns queries (dK / dV).  The thread's rows lie in 16-row block w (its warp), element 4 i + 2 hh + e in column
// block i / 2.
template <bool QROWS>
__device__ __forceinline__ uint32_t fa_sparse_vis_bits(uint32_t tm, int S, int r0, int c0, const Frag& f) {
  const int w = f.fr >> 4;
  const uint32_t nib = QROWS ? (tm >> (4 * w)) & 15u
                             : ((tm >> w) & 1u) | ((tm >> (w + 3)) & 2u) | ((tm >> (w + 6)) & 4u) | ((tm >> (w + 9)) & 8u);
  uint32_t bits = 0u;
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int row = r0 + f.fr + 8 * hh, col = c0 + 8 * i + f.fc + e;
        const bool vis = ((nib >> (i >> 1)) & 1u) && (QROWS ? col <= row && col < S : row <= col && col < S);
        bits |= (uint32_t)vis << (4 * i + 2 * hh + e);
      }
  return bits;
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------------
// forward: grid (query blocks, B * H); online softmax in the exp2 domain
// ------------------------------------------------------------------------------------------------------------------
template <int DH, bool DROP, bool LOCAL, bool AXIAL, bool CONV, bool SPARSE>
__global__ void __launch_bounds__(128, 1)
attn_fwd_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ out, float* __restrict__ lse, int S, int H,
                float scale, const db200_dropout dr, int radius, const FaAxial ax, const FaConv cv,
                const FaSparse sp) {
  static_assert(!(AXIAL && (DROP || LOCAL)), "axial layers have no dropout and no window");
  static_assert(!(CONV && (DROP || LOCAL || AXIAL)), "conv layers have no dropout, no window and no row map");
  static_assert(!(SPARSE && (DROP || LOCAL || AXIAL || CONV)), "block-sparse layers have no dropout and one mask");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t TILE = FA_ROWS * DH * 2;
  const uint32_t sQ = base, sK = base + TILE, sV = base + 2 * TILE;
  const int qb = blockIdx.x, b = blockIdx.y / H, h = blockIdx.y % H;
  const int q0 = qb * FA_ROWS;
  const long long ldq = 3LL * H * DH;
  const bf16* Q = qkv + (long long)b * S * ldq + (long long)h * DH;
  const Frag f;
  const float sl2 = scale * kLog2e;

  if constexpr (AXIAL) fa_load_tile_axial<DH>(sQ, Q, ldq, ax, S, q0);
  else fa_load_tile<DH>(sQ, Q + q0 * ldq, ldq, S - q0);
  float o[DH / 2], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
  int jt = 0, js = 0, slo[2] = {0, 0};  // AXIAL: key blocks and the segment start of each query row
  int qr[2] = {0, 0}, qc[2] = {0, 0};   // CONV: grid row / column of each query row
  if constexpr (AXIAL) {
    fa_axial_key_blocks(ax, qb, jt, js);
    slo[0] = fa_axial_seg_start(ax, q0 + f.fr);
    slo[1] = fa_axial_seg_start(ax, q0 + f.fr + 8);
  }
  if constexpr (CONV) {
    fa_conv_key_blocks(cv, qb, jt, js);
    fa_conv_rc(cv, q0 + f.fr, qr[0], qc[0]);
    fa_conv_rc(cv, q0 + f.fr + 8, qr[1], qc[1]);
  }
  const int j0 = SPARSE  ? fa_sparse_next_key(sp, qb, -1)
               : LOCAL ? max(0, q0 - radius + 1) / FA_ROWS
                       : ((AXIAL || CONV) && jt == 0 ? js : 0);
  for (int j = j0; j <= qb;
       j = SPARSE ? fa_sparse_next_key(sp, qb, j) : (AXIAL || CONV) ? fa_axial_next(j, jt, js) : j + 1) {
    const int k0 = j * FA_ROWS;
    __syncthreads();  // the previous block's K / V tiles are no longer read
    if constexpr (AXIAL) {
      fa_load_tile_axial<DH>(sK, Q + (long long)H * DH, ldq, ax, S, k0);
      fa_load_tile_axial<DH>(sV, Q + 2LL * H * DH, ldq, ax, S, k0);
    } else {
      fa_load_tile<DH>(sK, Q + k0 * ldq + (long long)H * DH, ldq, S - k0);
      fa_load_tile<DH>(sV, Q + k0 * ldq + 2LL * H * DH, ldq, S - k0);
    }
    fa_tiles_ready();
    float s[32];
    fa_qk<DH>(s, sQ, sK);
    const uint32_t vb = CONV     ? fa_conv_vis_bits<true>(cv, S, q0, k0, qr, qc, f)
                        : SPARSE ? fa_sparse_vis_bits<true>(fa_sparse_tile(sp, qb, j), S, q0, k0, f)
                                 : 0u;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int row = q0 + f.fr + 8 * hh, col = k0 + 8 * i + f.fc + e;
          float& v = s[4 * i + 2 * hh + e];
          if constexpr (AXIAL) v = (col <= row && (col < ax.text_len || col >= slo[hh])) ? v * sl2 : -INFINITY;
          else if constexpr (CONV || SPARSE) v = ((vb >> (4 * i + 2 * hh + e)) & 1u) ? v * sl2 : -INFINITY;
          else v = (col <= row && col < S && (!LOCAL || col > row - radius)) ? v * sl2 : -INFINITY;
          mx[hh] = fmaxf(mx[hh], v);
        }
    float alpha[2], mb[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const float mn = fmaxf(m[hh], quad_max(mx[hh]));
      mb[hh] = mn == -INFINITY ? 0.f : mn;
      alpha[hh] = exp2f(m[hh] - mb[hh]);
      m[hh] = mn;
      l[hh] *= alpha[hh];
    }
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) {
      o[4 * i + 0] *= alpha[0]; o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
    }
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = s[4 * i + 2 * hh + e];
          v = exp2f(v - mb[hh]);
          l[hh] += v;
        }
    // l (hence lse) sums the undropped weights; dropout acts on the normalised weights, i.e. on P before PV
    if constexpr (DROP)
      fa_pv<DH, true>(o, s, sV, fa_keep_bits<true>(dr, b, h, H, (S + 1) >> 1, q0, k0, f), dr.scale);
    else
      fa_pv<DH>(o, s, sV);
  }
  float inv[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float tot = quad_sum(l[hh]);
    inv[hh] = tot > 0.f ? 1.f / tot : 0.f;
    const int row = AXIAL ? fa_axial_pos(ax, S, q0 + f.fr + 8 * hh) : q0 + f.fr + 8 * hh;
    if ((f.fc == 0) && row < S && (!AXIAL || row >= 0))
      lse[((long long)b * H + h) * S + row] = (m[hh] + log2f(tot)) * kLn2;
  }
  if constexpr (AXIAL)
    fa_store_rows_axial<DH>(out + (long long)b * S * H * DH + (long long)h * DH, (long long)H * DH, o, inv, ax, S, q0, f);
  else
    fa_store_rows<DH>(out + ((long long)b * S + q0) * H * DH + (long long)h * DH, (long long)H * DH, o, inv, S - q0, f);
}

// ------------------------------------------------------------------------------------------------------------------
// backward, dQ: grid (query blocks, B * H).  P = exp(scale S - lse), dS = P (dO V^T - delta), dQ = scale dS K
// ------------------------------------------------------------------------------------------------------------------
template <int DH, bool DROP, bool LOCAL, bool AXIAL, bool CONV, bool SPARSE>
__global__ void __launch_bounds__(128, 1)
attn_bwd_dq_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ dout, const float* __restrict__ lse,
                   const float* __restrict__ delta, bf16* __restrict__ dqkv, int S, int H, float scale,
                   const db200_dropout dr, int radius, const FaAxial ax, const FaConv cv, const FaSparse sp) {
  static_assert(!(AXIAL && (DROP || LOCAL)), "axial layers have no dropout and no window");
  static_assert(!(CONV && (DROP || LOCAL || AXIAL)), "conv layers have no dropout, no window and no row map");
  static_assert(!(SPARSE && (DROP || LOCAL || AXIAL || CONV)), "block-sparse layers have no dropout and one mask");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t TILE = FA_ROWS * DH * 2;
  const uint32_t sQ = base, sdO = base + TILE, sK = base + 2 * TILE, sV = base + 3 * TILE;
  const int qb = blockIdx.x, b = blockIdx.y / H, h = blockIdx.y % H;
  const int q0 = qb * FA_ROWS;
  const long long ldq = 3LL * H * DH, ldo = (long long)H * DH;
  const bf16* Q = qkv + (long long)b * S * ldq + (long long)h * DH;
  const Frag f;
  const float sl2 = scale * kLog2e;

  int slo[2] = {0, 0};  // AXIAL: segment start of each query row
  if constexpr (AXIAL) {
    fa_load_tile_axial<DH>(sQ, Q, ldq, ax, S, q0);
    fa_load_tile_axial<DH>(sdO, dout + (long long)b * S * ldo + (long long)h * DH, ldo, ax, S, q0);
  } else {
    fa_load_tile<DH>(sQ, Q + q0 * ldq, ldq, S - q0);
    fa_load_tile<DH>(sdO, dout + ((long long)b * S + q0) * ldo + (long long)h * DH, ldo, S - q0);
  }
  float lse2[2], dl[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = q0 + f.fr + 8 * hh;
    if constexpr (AXIAL) {
      // an absent row gets P = 0 (lse = +inf) and dS = 0
      const int p = fa_axial_pos(ax, S, row);
      const long long ix = ((long long)b * H + h) * S + (p >= 0 ? p : 0);
      lse2[hh] = p >= 0 ? lse[ix] * kLog2e : INFINITY;
      dl[hh] = p >= 0 ? delta[ix] : 0.f;
      slo[hh] = fa_axial_seg_start(ax, row);
    } else {
      const long long ix = ((long long)b * H + h) * S + (row < S ? row : S - 1);
      lse2[hh] = lse[ix] * kLog2e;
      dl[hh] = delta[ix];
    }
  }
  float dq[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) dq[i] = 0.f;
  int jt = 0, js = 0, qr[2] = {0, 0}, qc[2] = {0, 0};  // CONV: grid row / column of each query row
  if constexpr (AXIAL) fa_axial_key_blocks(ax, qb, jt, js);
  if constexpr (CONV) {
    fa_conv_key_blocks(cv, qb, jt, js);
    fa_conv_rc(cv, q0 + f.fr, qr[0], qc[0]);
    fa_conv_rc(cv, q0 + f.fr + 8, qr[1], qc[1]);
  }
  const int j0 = SPARSE  ? fa_sparse_next_key(sp, qb, -1)
               : LOCAL ? max(0, q0 - radius + 1) / FA_ROWS
                       : ((AXIAL || CONV) && jt == 0 ? js : 0);
  for (int j = j0; j <= qb;
       j = SPARSE ? fa_sparse_next_key(sp, qb, j) : (AXIAL || CONV) ? fa_axial_next(j, jt, js) : j + 1) {
    const int k0 = j * FA_ROWS;
    __syncthreads();
    if constexpr (AXIAL) {
      fa_load_tile_axial<DH>(sK, Q + (long long)H * DH, ldq, ax, S, k0);
      fa_load_tile_axial<DH>(sV, Q + 2LL * H * DH, ldq, ax, S, k0);
    } else {
      fa_load_tile<DH>(sK, Q + k0 * ldq + (long long)H * DH, ldq, S - k0);
      fa_load_tile<DH>(sV, Q + k0 * ldq + 2LL * H * DH, ldq, S - k0);
    }
    fa_tiles_ready();
    float s[32], dp[32];
    fa_qk<DH>(s, sQ, sK);
    fa_qk<DH>(dp, sdO, sV);
    // dropout: dS = P (dP keep scale - delta)
    const uint32_t kb = DROP ? fa_keep_bits<true>(dr, b, h, H, (S + 1) >> 1, q0, k0, f) : 0u;
    const uint32_t vb = CONV     ? fa_conv_vis_bits<true>(cv, S, q0, k0, qr, qc, f)
                        : SPARSE ? fa_sparse_vis_bits<true>(fa_sparse_tile(sp, qb, j), S, q0, k0, f)
                                 : 0u;
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int row = q0 + f.fr + 8 * hh, col = k0 + 8 * i + f.fc + e;
          const int x = 4 * i + 2 * hh + e;
          const bool vis = AXIAL ? col <= row && (col < ax.text_len || col >= slo[hh])
                         : (CONV || SPARSE) ? ((vb >> x) & 1u) != 0u
                                 : col <= row && col < S && row < S && (!LOCAL || col > row - radius);
          const float p = vis ? exp2f(s[x] * sl2 - lse2[hh]) : 0.f;
          s[x] = p * ((DROP ? dp[x] * fa_keep_mul(kb, x, dr.scale) : dp[x]) - dl[hh]);
        }
    fa_pv<DH>(dq, s, sK);
  }
  const float mul[2] = {scale, scale};
  if constexpr (AXIAL) fa_store_rows_axial<DH>(dqkv + (long long)b * S * ldq + (long long)h * DH, ldq, dq, mul, ax, S, q0, f);
  else fa_store_rows<DH>(dqkv + ((long long)b * S + q0) * ldq + (long long)h * DH, ldq, dq, mul, S - q0, f);
}

// ------------------------------------------------------------------------------------------------------------------
// backward, dK / dV: grid (key blocks, B * H), transposed products so that the key index is the accumulator row.
//   P^T = exp(scale K Q^T - lse), dV = P^T dO, dS^T = P^T (V dO^T - delta), dK = scale dS^T Q
// ------------------------------------------------------------------------------------------------------------------
template <int DH, bool DROP, bool LOCAL, bool AXIAL, bool CONV, bool SPARSE>
__global__ void __launch_bounds__(128, 1)
attn_bwd_dkv_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ dout, const float* __restrict__ lse,
                    const float* __restrict__ delta, bf16* __restrict__ dqkv, int S, int H, float scale,
                    const db200_dropout dr, int radius, const FaAxial ax, const FaConv cv, const FaSparse sp) {
  static_assert(!(AXIAL && (DROP || LOCAL)), "axial layers have no dropout and no window");
  static_assert(!(CONV && (DROP || LOCAL || AXIAL)), "conv layers have no dropout, no window and no row map");
  static_assert(!(SPARSE && (DROP || LOCAL || AXIAL || CONV)), "block-sparse layers have no dropout and one mask");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t TILE = FA_ROWS * DH * 2;
  const uint32_t sK = base, sV = base + TILE, sQ = base + 2 * TILE, sdO = base + 3 * TILE;
  float* s_lse = reinterpret_cast<float*>(smem_raw + (base + 4 * TILE - smem_u32(smem_raw)));
  float* s_dl = s_lse + FA_ROWS;
  const int kb = blockIdx.x, b = blockIdx.y / H, h = blockIdx.y % H;
  const int k0 = kb * FA_ROWS;
  const long long ldq = 3LL * H * DH, ldo = (long long)H * DH;
  const bf16* Q = qkv + (long long)b * S * ldq + (long long)h * DH;
  const Frag f;
  const float sl2 = scale * kLog2e;
  // LOCAL: the last query that sees key k0 + 63 is k0 + 62 + radius
  // AXIAL: fa_axial_query_end; a key row sees the queries up to the end of its segment (text keys: every later one)
  // CONV: fa_conv_query_end
  const int nqb = AXIAL ? fa_axial_query_end(ax, kb)
                : CONV  ? fa_conv_query_end(cv, S, kb)
                : LOCAL ? min((S + FA_ROWS - 1) / FA_ROWS, (int)(((long long)k0 + 62 + radius) / FA_ROWS) + 1)
                        : (S + FA_ROWS - 1) / FA_ROWS;
  int kr[2] = {0, 0}, kc[2] = {0, 0};  // CONV: grid row / column of each key row
  if constexpr (CONV) {
    fa_conv_rc(cv, k0 + f.fr, kr[0], kc[0]);
    fa_conv_rc(cv, k0 + f.fr + 8, kr[1], kc[1]);
  }
  int kend[2] = {0, 0};
  if constexpr (AXIAL) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int key = k0 + f.fr + 8 * hh;
      kend[hh] = key < ax.text_len ? INT_MAX : fa_axial_seg_start(ax, key) + ax.grid_w - 1;
    }
    fa_load_tile_axial<DH>(sK, Q + (long long)H * DH, ldq, ax, S, k0);
    fa_load_tile_axial<DH>(sV, Q + 2LL * H * DH, ldq, ax, S, k0);
  } else {
    fa_load_tile<DH>(sK, Q + k0 * ldq + (long long)H * DH, ldq, S - k0);
    fa_load_tile<DH>(sV, Q + k0 * ldq + 2LL * H * DH, ldq, S - k0);
  }
  float dk[DH / 2], dv[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) { dk[i] = 0.f; dv[i] = 0.f; }
  for (int i = SPARSE ? fa_sparse_next_query(sp, kb, kb - 1, nqb) : kb; i < nqb;
       i = SPARSE ? fa_sparse_next_query(sp, kb, i, nqb) : i + 1) {
    const int q0 = i * FA_ROWS;
    __syncthreads();
    if constexpr (AXIAL) {
      fa_load_tile_axial<DH>(sQ, Q, ldq, ax, S, q0);
      fa_load_tile_axial<DH>(sdO, dout + (long long)b * S * ldo + (long long)h * DH, ldo, ax, S, q0);
      if (threadIdx.x < FA_ROWS) {  // an absent query gets P = 0 (lse = +inf) and dS = 0
        const int p = fa_axial_pos(ax, S, q0 + threadIdx.x);
        const long long ix = ((long long)b * H + h) * S + (p >= 0 ? p : 0);
        s_lse[threadIdx.x] = p >= 0 ? lse[ix] * kLog2e : INFINITY;
        s_dl[threadIdx.x] = p >= 0 ? delta[ix] : 0.f;
      }
    } else {
      fa_load_tile<DH>(sQ, Q + q0 * ldq, ldq, S - q0);
      fa_load_tile<DH>(sdO, dout + ((long long)b * S + q0) * ldo + (long long)h * DH, ldo, S - q0);
      if (threadIdx.x < FA_ROWS) {
        const int q = q0 + threadIdx.x;
        const long long ix = ((long long)b * H + h) * S + (q < S ? q : S - 1);
        s_lse[threadIdx.x] = lse[ix] * kLog2e;
        s_dl[threadIdx.x] = delta[ix];
      }
    }
    fa_tiles_ready();
    float st[32], dpt[32];
    fa_qk<DH>(st, sK, sQ);
    const uint32_t vb = CONV     ? fa_conv_vis_bits<false>(cv, S, k0, q0, kr, kc, f)
                        : SPARSE ? fa_sparse_vis_bits<false>(fa_sparse_tile(sp, i, kb), S, k0, q0, f)
                                 : 0u;
#pragma unroll
    for (int ii = 0; ii < 8; ++ii)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = k0 + f.fr + 8 * hh, cq = 8 * ii + f.fc + e, q = q0 + cq;
          const int x = 4 * ii + 2 * hh + e;
          const bool vis = AXIAL ? key <= q && (key < ax.text_len || q <= kend[hh])
                         : (CONV || SPARSE) ? ((vb >> x) & 1u) != 0u
                                 : key <= q && q < S && key < S && (!LOCAL || key > q - radius);
          st[x] = vis ? exp2f(st[x] * sl2 - s_lse[cq]) : 0.f;
        }
    // dropout: dV += (P keep scale)^T dO,  dS = P (dP keep scale - delta)
    const uint32_t kb = DROP ? fa_keep_bits<false>(dr, b, h, H, (S + 1) >> 1, k0, q0, f) : 0u;
    if constexpr (DROP) fa_pv<DH, true>(dv, st, sdO, kb, dr.scale);
    else fa_pv<DH>(dv, st, sdO);
    fa_qk<DH>(dpt, sV, sdO);
#pragma unroll
    for (int ii = 0; ii < 8; ++ii)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * ii + 2 * hh + e;
          st[x] = st[x] * ((DROP ? dpt[x] * fa_keep_mul(kb, x, dr.scale) : dpt[x]) - s_dl[8 * ii + f.fc + e]);
        }
    fa_pv<DH>(dk, st, sQ);
  }
  const float one[2] = {1.f, 1.f}, mul[2] = {scale, scale};
  if constexpr (AXIAL) {
    bf16* dst = dqkv + (long long)b * S * ldq + (long long)h * DH;
    fa_store_rows_axial<DH>(dst + (long long)H * DH, ldq, dk, mul, ax, S, k0, f);
    fa_store_rows_axial<DH>(dst + 2LL * H * DH, ldq, dv, one, ax, S, k0, f);
  } else {
    bf16* dst = dqkv + ((long long)b * S + k0) * ldq + (long long)h * DH;
    fa_store_rows<DH>(dst + (long long)H * DH, ldq, dk, mul, S - k0, f);
    fa_store_rows<DH>(dst + 2LL * H * DH, ldq, dv, one, S - k0, f);
  }
}

// AXIAL: the grid covers ax.rows kernel-order rows instead of S
template <int DH, bool DROP, bool LOCAL = false, bool AXIAL = false, bool CONV = false, bool SPARSE = false>
static int fa_fwd(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, float scale,
                  const db200_dropout& dr, int radius = 0, const FaAxial& ax = FaAxial{},
                  const FaConv& cv = FaConv{}, const FaSparse& sp = FaSparse{}) {
  constexpr size_t smem = fa_smem<DH>(3);
  static const cudaError_t attr_rc = cudaFuncSetAttribute(attn_fwd_kernel<DH, DROP, LOCAL, AXIAL, CONV, SPARSE>,
                                                          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  DB200_CUDA(attr_rc);
  const dim3 grid(((AXIAL ? ax.rows : S) + FA_ROWS - 1) / FA_ROWS, B * H);
  attn_fwd_kernel<DH, DROP, LOCAL, AXIAL, CONV, SPARSE><<<grid, 128, smem, stream>>>(
      (const bf16*)qkv, (bf16*)out, lse, S, H, scale, dr, radius, ax, cv, sp);
  return check_launch("attn_fwd_kernel");
}

template <int DH, bool DROP, bool LOCAL = false, bool AXIAL = false, bool CONV = false, bool SPARSE = false>
static int fa_bwd(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                  void* dqkv, int B, int S, int H, float scale, const db200_dropout& dr, int radius = 0,
                  const FaAxial& ax = FaAxial{}, const FaConv& cv = FaConv{}, const FaSparse& sp = FaSparse{}) {
  constexpr size_t smem = fa_smem<DH>(4);
  static const cudaError_t rc1 = cudaFuncSetAttribute(attn_bwd_dq_kernel<DH, DROP, LOCAL, AXIAL, CONV, SPARSE>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  static const cudaError_t rc2 = cudaFuncSetAttribute(attn_bwd_dkv_kernel<DH, DROP, LOCAL, AXIAL, CONV, SPARSE>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  DB200_CUDA(rc1);
  DB200_CUDA(rc2);
  const dim3 grid(((AXIAL ? ax.rows : S) + FA_ROWS - 1) / FA_ROWS, B * H);
  attn_bwd_dq_kernel<DH, DROP, LOCAL, AXIAL, CONV, SPARSE><<<grid, 128, smem, stream>>>(
      (const bf16*)qkv, (const bf16*)dout, lse, delta, (bf16*)dqkv, S, H, scale, dr, radius, ax, cv, sp);
  int rc = check_launch("attn_bwd_dq_kernel");
  if (rc != DB200_OK) return rc;
  attn_bwd_dkv_kernel<DH, DROP, LOCAL, AXIAL, CONV, SPARSE><<<grid, 128, smem, stream>>>(
      (const bf16*)qkv, (const bf16*)dout, lse, delta, (bf16*)dqkv, S, H, scale, dr, radius, ax, cv, sp);
  return check_launch("attn_bwd_dkv_kernel");
}

// drop == NULL (or threshold 0): the kernels without dropout
int attn_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, int dh,
                    float scale, const db200_dropout* drop) {
  const db200_dropout none{};
  if (dropout_active(drop))
    return dh == 128 ? fa_fwd<128, true>(stream, qkv, out, lse, B, S, H, scale, *drop)
                     : fa_fwd<64, true>(stream, qkv, out, lse, B, S, H, scale, *drop);
  return dh == 128 ? fa_fwd<128, false>(stream, qkv, out, lse, B, S, H, scale, none)
                   : fa_fwd<64, false>(stream, qkv, out, lse, B, S, H, scale, none);
}

int attn_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                    void* dqkv, int B, int S, int H, int dh, float scale, const db200_dropout* drop) {
  const db200_dropout none{};
  if (dropout_active(drop))
    return dh == 128 ? fa_bwd<128, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, *drop)
                     : fa_bwd<64, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, *drop);
  return dh == 128 ? fa_bwd<128, false>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none)
                   : fa_bwd<64, false>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none);
}

// sliding window of `radius` keys (radius >= 1); no attention dropout (local layers have none)
int attn_local_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, int dh,
                          int radius, float scale) {
  const db200_dropout none{};
  return dh == 128 ? fa_fwd<128, false, true>(stream, qkv, out, lse, B, S, H, scale, none, radius)
                   : fa_fwd<64, false, true>(stream, qkv, out, lse, B, S, H, scale, none, radius);
}

int attn_local_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                          void* dqkv, int B, int S, int H, int dh, int radius, float scale) {
  const db200_dropout none{};
  return dh == 128 ? fa_bwd<128, false, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none, radius)
                   : fa_bwd<64, false, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none, radius);
}

// kernel-order rows of an axial layer of length S: S for a row layer (or without image rows); for a column layer, one
// past the largest u = c W + r of the present image tokens k = r W + c < S - TL
static int axial_rows(int S, int text_len, int grid_w, int axis) {
  const int n = S - text_len;
  if (!axis || n <= 0) return S;
  const int umax = n >= grid_w ? (grid_w - 1) * grid_w + (n - grid_w) / grid_w : (n - 1) * grid_w;
  return text_len + umax + 1;
}

// row (axis 0) or column (axis 1) attention over a text prefix of text_len and a grid_w x grid_w image; no dropout
int attn_axial_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, int dh,
                          int text_len, int grid_w, int axis, float scale) {
  const db200_dropout none{};
  const FaAxial ax{text_len, grid_w, axis, axial_rows(S, text_len, grid_w, axis)};
  return dh == 128 ? fa_fwd<128, false, false, true>(stream, qkv, out, lse, B, S, H, scale, none, 0, ax)
                   : fa_fwd<64, false, false, true>(stream, qkv, out, lse, B, S, H, scale, none, 0, ax);
}

int attn_axial_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                          void* dqkv, int B, int S, int H, int dh, int text_len, int grid_w, int axis, float scale) {
  const db200_dropout none{};
  const FaAxial ax{text_len, grid_w, axis, axial_rows(S, text_len, grid_w, axis)};
  return dh == 128 ? fa_bwd<128, false, false, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none, 0, ax)
                   : fa_bwd<64, false, false, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none, 0, ax);
}

// convolutional attention (k x k window) over a text prefix of text_len and a grid_w x grid_w image; no dropout
int attn_conv_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H, int dh,
                         int text_len, int grid_w, int kernel, float scale) {
  const db200_dropout none{};
  const FaConv cv{text_len, grid_w, kernel};
  return dh == 128 ? fa_fwd<128, false, false, false, true>(stream, qkv, out, lse, B, S, H, scale, none, 0, {}, cv)
                   : fa_fwd<64, false, false, false, true>(stream, qkv, out, lse, B, S, H, scale, none, 0, {}, cv);
}

int attn_conv_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse, const float* delta,
                         void* dqkv, int B, int S, int H, int dh, int text_len, int grid_w, int kernel, float scale) {
  const db200_dropout none{};
  const FaConv cv{text_len, grid_w, kernel};
  return dh == 128
             ? fa_bwd<128, false, false, false, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none, 0, {}, cv)
             : fa_bwd<64, false, false, false, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale, none, 0, {}, cv);
}

// block-sparse attention over the tile masks of `mask` (row pitch `pitch`); no dropout
int attn_block_sparse_fwd_launch(cudaStream_t stream, const void* qkv, void* out, float* lse, int B, int S, int H,
                                 int dh, const uint16_t* mask, int pitch, float scale) {
  const db200_dropout none{};
  const FaSparse sp{mask, pitch};
  return dh == 128
             ? fa_fwd<128, false, false, false, false, true>(stream, qkv, out, lse, B, S, H, scale, none, 0, {}, {}, sp)
             : fa_fwd<64, false, false, false, false, true>(stream, qkv, out, lse, B, S, H, scale, none, 0, {}, {}, sp);
}

int attn_block_sparse_bwd_launch(cudaStream_t stream, const void* qkv, const void* dout, const float* lse,
                                 const float* delta, void* dqkv, int B, int S, int H, int dh, const uint16_t* mask,
                                 int pitch, float scale) {
  const db200_dropout none{};
  const FaSparse sp{mask, pitch};
  return dh == 128 ? fa_bwd<128, false, false, false, false, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale,
                                                                   none, 0, {}, {}, sp)
                   : fa_bwd<64, false, false, false, false, true>(stream, qkv, dout, lse, delta, dqkv, B, S, H, scale,
                                                                  none, 0, {}, {}, sp);
}

}  // namespace db200
