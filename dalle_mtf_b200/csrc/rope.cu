// Rotary position embeddings (extension; GPT-NeoX's rotate_half layout with partial rotary) on the fused q|k|v rows.
//
// A row of qkv is [3][H][dh] bf16 (q heads, k heads, v heads).  For every q and k head, the pair (x_j, x_{j+h}) of its
// first r dims (h = r / 2, j < h) is rotated by the angle p theta_j of the row's position p:
//   x_j'     = x_j c - x_{j+h} s,   x_{j+h}' = x_{j+h} c + x_j s,   c = cos(p theta_j), s = sin(p theta_j)
// (the backward applies the transpose: s -> -s).  Every product and sum is rounded on its own (__fmul_rn, __fadd_rn,
// __fsub_rn: no FMA contraction), so a float32 evaluation of the same expression reproduces the result bit for bit.
// v and the dims r .. dh-1 are not touched.  The table is fp32 [n_pos][2][h]: position p's h cosines, then its h sines.
// The kernels are HBM-bound in-place updates: 16-byte vectors when h % 8 == 0, one pair per thread otherwise.
//
// The same kernel, with IL set, applies DALLE-pytorch's rotary embedding (rotary_emb): interleaved pairs (x_2m,
// x_2m+1), m < h (h = 3 nf pairs), of every q, k AND v head (3H heads), each pair at its own angle of the row's table
// entry [2][h] (cosines, then sines; the text / row / column parts are laid out in the table, not here).  With 16-byte
// vectors (G = 4 pairs) the last group of a head may hold fewer than G pairs; it is done one pair at a time.
#include "common.cuh"

namespace db200 {

template <bool INV>
__device__ __forceinline__ void rope_pair(float a, float b, float c, float s, float& ao, float& bo) {
  if (!INV) {
    ao = __fsub_rn(__fmul_rn(a, c), __fmul_rn(b, s));
    bo = __fadd_rn(__fmul_rn(b, c), __fmul_rn(a, s));
  } else {
    ao = __fadd_rn(__fmul_rn(a, c), __fmul_rn(b, s));
    bo = __fsub_rn(__fmul_rn(b, c), __fmul_rn(a, s));
  }
}

// One work item: (row t, head hh of the 2H q|k heads (IL: the 3H q|k|v heads), group g of G pairs).  The row's position is *pos_dev when
// pos_dev is set, else pos when pos >= 0, else t mod S; a position outside [0, n_pos) leaves the row unchanged.
template <int G, bool INV, bool IL = false>
__global__ void __launch_bounds__(256)
rope_kernel(bf16* __restrict__ qkv, const float* __restrict__ table, long long rows, int S, int H, int dh, int h,
            int pos, const int* __restrict__ pos_dev, int n_pos) {
  const int groups = IL ? (h + G - 1) / G : h / G;
  const long long per_row = (long long)(IL ? 3 : 2) * H * groups;
  const long long total = rows * per_row;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const bool by_row = !pos_dev && pos < 0;
  const int fixed = pos_dev ? *pos_dev : pos;
  const long long row_len = (long long)3 * H * dh;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += stride) {
    const long long t = i / per_row;
    const int rem = (int)(i - t * per_row);
    const int hh = rem / groups;
    const int j0 = (rem - hh * groups) * G;
    const int p = by_row ? (int)(t % S) : fixed;
    if (p < 0 || p >= n_pos) continue;
    bf16* x = qkv + t * row_len + (long long)hh * dh + (IL ? 2 * j0 : j0);
    const float* cs = table + (long long)p * 2 * h + j0;
    if constexpr (IL) {
      // the table rows are h floats long (h odd for dh 128), so cos / sin are read as scalars: they are L1-resident
      __nv_bfloat162* px = reinterpret_cast<__nv_bfloat162*>(x);
      const int n = h - j0 < G ? h - j0 : G;
      if (G == 4 && n == G) {
        uint4 v = *reinterpret_cast<const uint4*>(x);
        __nv_bfloat162* pv = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
        for (int k = 0; k < G; ++k) {
          const float2 a = __bfloat1622float2(pv[k]);
          float2 o;
          rope_pair<INV>(a.x, a.y, cs[k], cs[h + k], o.x, o.y);
          pv[k] = __float22bfloat162_rn(o);
        }
        *reinterpret_cast<uint4*>(x) = v;
      } else {
        for (int k = 0; k < n; ++k) {
          const float2 a = __bfloat1622float2(px[k]);
          float2 o;
          rope_pair<INV>(a.x, a.y, cs[k], cs[h + k], o.x, o.y);
          px[k] = __float22bfloat162_rn(o);
        }
      }
    } else if constexpr (G == 8) {
      uint4 va = *reinterpret_cast<const uint4*>(x);
      uint4 vb = *reinterpret_cast<const uint4*>(x + h);
      const float4 c0 = *reinterpret_cast<const float4*>(cs), c1 = *reinterpret_cast<const float4*>(cs + 4);
      const float4 s0 = *reinterpret_cast<const float4*>(cs + h), s1 = *reinterpret_cast<const float4*>(cs + h + 4);
      const float c[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      const float s[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
      __nv_bfloat162* pa = reinterpret_cast<__nv_bfloat162*>(&va);
      __nv_bfloat162* pb = reinterpret_cast<__nv_bfloat162*>(&vb);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 a = __bfloat1622float2(pa[k]), b = __bfloat1622float2(pb[k]);
        float2 ao, bo;
        rope_pair<INV>(a.x, b.x, c[2 * k], s[2 * k], ao.x, bo.x);
        rope_pair<INV>(a.y, b.y, c[2 * k + 1], s[2 * k + 1], ao.y, bo.y);
        pa[k] = __float22bfloat162_rn(ao);
        pb[k] = __float22bfloat162_rn(bo);
      }
      *reinterpret_cast<uint4*>(x) = va;
      *reinterpret_cast<uint4*>(x + h) = vb;
    } else {
      float ao, bo;
      rope_pair<INV>(__bfloat162float(x[0]), __bfloat162float(x[h]), cs[0], cs[h], ao, bo);
      x[0] = __float2bfloat16_rn(ao);
      x[h] = __float2bfloat16_rn(bo);
    }
  }
}

static int rope_grid(long long work) {
  const long long cap = (long long)sm_count() * 16;
  const long long blocks = (work + 255) / 256;
  return (int)(blocks < 1 ? 1 : (blocks < cap ? blocks : cap));
}

// Shared argument checks and launch.  S: the period of t -> position (pos < 0, no pos_dev) or the table's length
// (decode: the position must lie in [0, S)).
static int rope_launch(cudaStream_t stream, void* qkv, const float* table, int rows, int S, int H, int dh, int r,
                       int pos, const int32_t* pos_dev, bool inv, const char* what) {
  DB200_REQUIRE(qkv && table, DB200_E_INVALID, "%s: NULL pointer", what);
  DB200_REQUIRE(rows > 0 && S > 0 && H > 0 && dh > 0, DB200_E_INVALID,
                "%s: need rows, S, H and dh > 0 (got rows=%d S=%d H=%d dh=%d)", what, rows, S, H, dh);
  DB200_REQUIRE(r >= 2 && r <= dh && r % 2 == 0, DB200_E_INVALID,
                "%s: rotary_dim must be even with 2 <= r <= dh (got r=%d dh=%d)", what, r, dh);
  const int h = r / 2;
  const bool vec = h % 8 == 0 && dh % 8 == 0;
  DB200_REQUIRE(!vec || (aligned16(qkv) && aligned16(table)), DB200_E_ALIGN,
                "%s: qkv and the table must be 16-byte aligned", what);
  const long long work = (long long)rows * 2 * H * (vec ? h / 8 : h);
  const int grid = rope_grid(work);
  bf16* x = static_cast<bf16*>(qkv);
  if (vec) {
    if (inv) rope_kernel<8, true><<<grid, 256, 0, stream>>>(x, table, rows, S, H, dh, h, pos, pos_dev, S);
    else     rope_kernel<8, false><<<grid, 256, 0, stream>>>(x, table, rows, S, H, dh, h, pos, pos_dev, S);
  } else {
    if (inv) rope_kernel<1, true><<<grid, 256, 0, stream>>>(x, table, rows, S, H, dh, h, pos, pos_dev, S);
    else     rope_kernel<1, false><<<grid, 256, 0, stream>>>(x, table, rows, S, H, dh, h, pos, pos_dev, S);
  }
  return check_launch(what);
}

// rotary_emb: pairs = 3 nf interleaved pairs of every q, k and v head; the table is fp32 [S][2][pairs].
static int rope_emb_launch(cudaStream_t stream, void* qkv, const float* table, int rows, int S, int H, int dh,
                           int pairs, int pos, const int32_t* pos_dev, bool inv, const char* what) {
  DB200_REQUIRE(qkv && table, DB200_E_INVALID, "%s: NULL pointer", what);
  DB200_REQUIRE(rows > 0 && S > 0 && H > 0 && dh > 0 && dh % 2 == 0, DB200_E_INVALID,
                "%s: need rows, S, H > 0 and an even dh > 0 (got rows=%d S=%d H=%d dh=%d)", what, rows, S, H, dh);
  DB200_REQUIRE(pairs >= 1 && 2 * pairs <= dh, DB200_E_INVALID, "%s: need 1 <= pairs <= dh / 2 (got pairs=%d dh=%d)",
                what, pairs, dh);
  const bool vec = dh % 8 == 0;
  DB200_REQUIRE(vec ? aligned16(qkv) : (reinterpret_cast<uintptr_t>(qkv) % 4 == 0), DB200_E_ALIGN,
                "%s: qkv must be %d-byte aligned", what, vec ? 16 : 4);
  DB200_REQUIRE(reinterpret_cast<uintptr_t>(table) % 4 == 0, DB200_E_ALIGN, "%s: the table must be 4-byte aligned",
                what);
  const int G = vec ? 4 : 1;
  const long long work = (long long)rows * 3 * H * ((pairs + G - 1) / G);
  const int grid = rope_grid(work);
  bf16* x = static_cast<bf16*>(qkv);
  if (vec) {
    if (inv) rope_kernel<4, true, true><<<grid, 256, 0, stream>>>(x, table, rows, S, H, dh, pairs, pos, pos_dev, S);
    else     rope_kernel<4, false, true><<<grid, 256, 0, stream>>>(x, table, rows, S, H, dh, pairs, pos, pos_dev, S);
  } else {
    if (inv) rope_kernel<1, true, true><<<grid, 256, 0, stream>>>(x, table, rows, S, H, dh, pairs, pos, pos_dev, S);
    else     rope_kernel<1, false, true><<<grid, 256, 0, stream>>>(x, table, rows, S, H, dh, pairs, pos, pos_dev, S);
  }
  return check_launch(what);
}

}  // namespace db200

using namespace db200;

extern "C" int db200_rope_fwd(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S, int H, int dh,
                              int r) {
  return rope_launch(reinterpret_cast<cudaStream_t>(stream), qkv_bf16, table, rows, S, H, dh, r, -1, nullptr, false,
                     "rope_fwd");
}

extern "C" int db200_rope_bwd(db200_stream_t stream, void* dqkv_bf16, const float* table, int rows, int S, int H,
                              int dh, int r) {
  return rope_launch(reinterpret_cast<cudaStream_t>(stream), dqkv_bf16, table, rows, S, H, dh, r, -1, nullptr, true,
                     "rope_bwd");
}

extern "C" int db200_rope_decode(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S, int H,
                                 int dh, int r, int pos) {
  DB200_REQUIRE(pos >= 0 && pos < S, DB200_E_INVALID, "rope_decode: position %d outside [0, %d)", pos, S);
  return rope_launch(reinterpret_cast<cudaStream_t>(stream), qkv_bf16, table, rows, S, H, dh, r, pos, nullptr, false,
                     "rope_decode");
}

extern "C" int db200_rope_decode_dev(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S, int H,
                                     int dh, int r, const int32_t* pos_dev) {
  DB200_REQUIRE(pos_dev, DB200_E_INVALID, "rope_decode_dev: NULL pos_dev");
  return rope_launch(reinterpret_cast<cudaStream_t>(stream), qkv_bf16, table, rows, S, H, dh, r, -1, pos_dev, false,
                     "rope_decode_dev");
}

extern "C" int db200_rope_emb_fwd(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S, int H,
                                  int dh, int pairs) {
  return rope_emb_launch(reinterpret_cast<cudaStream_t>(stream), qkv_bf16, table, rows, S, H, dh, pairs, -1, nullptr,
                         false, "rope_emb_fwd");
}

extern "C" int db200_rope_emb_bwd(db200_stream_t stream, void* dqkv_bf16, const float* table, int rows, int S, int H,
                                  int dh, int pairs) {
  return rope_emb_launch(reinterpret_cast<cudaStream_t>(stream), dqkv_bf16, table, rows, S, H, dh, pairs, -1, nullptr,
                         true, "rope_emb_bwd");
}

extern "C" int db200_rope_emb_decode(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S, int H,
                                     int dh, int pairs, int pos) {
  DB200_REQUIRE(pos >= 0 && pos < S, DB200_E_INVALID, "rope_emb_decode: position %d outside [0, %d)", pos, S);
  return rope_emb_launch(reinterpret_cast<cudaStream_t>(stream), qkv_bf16, table, rows, S, H, dh, pairs, pos, nullptr,
                         false, "rope_emb_decode");
}

extern "C" int db200_rope_emb_decode_dev(db200_stream_t stream, void* qkv_bf16, const float* table, int rows, int S,
                                         int H, int dh, int pairs, const int32_t* pos_dev) {
  DB200_REQUIRE(pos_dev, DB200_E_INVALID, "rope_emb_decode_dev: NULL pos_dev");
  return rope_emb_launch(reinterpret_cast<cudaStream_t>(stream), qkv_bf16, table, rows, S, H, dh, pairs, -1, pos_dev,
                         false, "rope_emb_decode_dev");
}
