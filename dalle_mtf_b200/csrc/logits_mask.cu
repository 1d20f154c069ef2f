// Modality logits mask (extension): the row partition around the two windowed vocabulary products.
//
// Row p of a sequence is a text row iff p < text_rows (= text_seq_len - 1: its target is a text token); it normalises
// over vocabulary ids [0, image_offset).  The other rows are image rows (targets: image codes and EOS) and normalise
// over [image_offset, V).  The training step gathers each class into a contiguous block, runs the unchanged wgmma
// GEMMs and CE epilogues on each block over its window of the vocabulary, and scatters the results back into [B * S]
// row order.
// Both kernels are HBM-bound copies with 16-byte vectors; no data reuse.
#include "common.cuh"

namespace db200 {

// Grid-stride loops over three ranges: the d / 8 16-byte vectors of every row of hf, the T labels and the image
// window's n_bias bias entries.
__global__ void __launch_bounds__(256)
logits_mask_partition_kernel(const uint4* __restrict__ hf, const int* __restrict__ labels,
                             const float* __restrict__ bias, uint4* __restrict__ hf_text, uint4* __restrict__ hf_image,
                             int* __restrict__ labels_text, int* __restrict__ labels_image,
                             float* __restrict__ bias_image, long long T, int S, int text_rows, int d16, int c0,
                             int image_offset, int V, int n_bias) {
  const int image_rows = S - text_rows;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long total = T * d16;
  for (long long i = i0; i < total; i += stride) {
    const long long t = i / d16;
    const int c = (int)(i - t * d16);
    const long long b = t / S;
    const int p = (int)(t - b * S);
    const uint4 v = hf[i];
    if (p < text_rows) hf_text[(b * text_rows + p) * d16 + c] = v;
    else               hf_image[(b * image_rows + (p - text_rows)) * d16 + c] = v;
  }
  for (long long t = i0; t < T; t += stride) {
    const long long b = t / S;
    const int p = (int)(t - b * S);
    const int l = labels[t];
    if (p < text_rows) labels_text[b * text_rows + p] = l;
    else               labels_image[b * image_rows + (p - text_rows)] = l - c0;
  }
  for (long long j = i0; j < n_bias; j += stride) {
    const int col = c0 + (int)j;
    bias_image[j] = col < image_offset ? -INFINITY : (col < V ? bias[col] : 0.f);
  }
}

// The inverse row map: dx (bf16 [T][d]) from the two blocks' dgrads, loss_rows ([T]) from the two blocks' row losses.
__global__ void __launch_bounds__(256)
logits_mask_scatter_kernel(const uint4* __restrict__ dx_text, const uint4* __restrict__ dx_image,
                           uint4* __restrict__ dx, const float* __restrict__ loss_text,
                           const float* __restrict__ loss_image, float* __restrict__ loss_rows, long long T, int S,
                           int text_rows, int d16) {
  const int image_rows = S - text_rows;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (dx) {
    const long long total = T * d16;
    for (long long i = i0; i < total; i += stride) {
      const long long t = i / d16;
      const int c = (int)(i - t * d16);
      const long long b = t / S;
      const int p = (int)(t - b * S);
      dx[i] = p < text_rows ? dx_text[(b * text_rows + p) * d16 + c]
                            : dx_image[(b * image_rows + (p - text_rows)) * d16 + c];
    }
  }
  if (loss_rows) {
    for (long long t = i0; t < T; t += stride) {
      const long long b = t / S;
      const int p = (int)(t - b * S);
      loss_rows[t] = p < text_rows ? loss_text[b * text_rows + p] : loss_image[b * image_rows + (p - text_rows)];
    }
  }
}

static int grid_for(long long work) {
  const long long cap = (long long)sm_count() * 16;
  const long long blocks = (work + 255) / 256;
  return (int)(blocks < 1 ? 1 : (blocks < cap ? blocks : cap));
}

}  // namespace db200

using namespace db200;

extern "C" int db200_logits_mask_partition(db200_stream_t stream_, const void* hf, const int32_t* labels,
                                           const float* bias, void* hf_text, void* hf_image, int32_t* labels_text,
                                           int32_t* labels_image, float* bias_image, int B, int S, int text_rows, int d,
                                           int c0, int image_offset, int V) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && S > 0 && text_rows >= 0 && text_rows < S && d > 0 && d % 8 == 0, DB200_E_INVALID,
                "logits_mask_partition: need B, S > 0, 0 <= text_rows < S and d a positive multiple of 8 (got B=%d "
                "S=%d text_rows=%d d=%d)", B, S, text_rows, d);
  DB200_REQUIRE(c0 >= 0 && c0 % 8 == 0 && c0 <= image_offset && image_offset < V, DB200_E_INVALID,
                "logits_mask_partition: need 0 <= c0 <= image_offset < V with c0 %% 8 == 0 (got c0=%d image_offset=%d "
                "V=%d)", c0, image_offset, V);
  DB200_REQUIRE(hf && labels && bias && hf_image && labels_image && bias_image &&
                    (text_rows == 0 || (hf_text && labels_text)),
                DB200_E_INVALID, "logits_mask_partition: NULL pointer");
  DB200_REQUIRE(aligned16(hf) && aligned16(hf_image) && (text_rows == 0 || aligned16(hf_text)), DB200_E_ALIGN,
                "logits_mask_partition: hf and its blocks must be 16-byte aligned");
  const long long T = (long long)B * S;
  const int d16 = d / 8;
  const int n_bias = (V - c0 + 7) / 8 * 8;
  logits_mask_partition_kernel<<<grid_for(T * d16), 256, 0, stream>>>(
      static_cast<const uint4*>(hf), labels, bias, static_cast<uint4*>(hf_text), static_cast<uint4*>(hf_image),
      labels_text, labels_image, bias_image, T, S, text_rows, d16, c0, image_offset, V, n_bias);
  return check_launch("logits_mask_partition_kernel");
}

extern "C" int db200_logits_mask_scatter(db200_stream_t stream_, const void* dx_text, const void* dx_image, void* dx,
                                         const float* loss_text, const float* loss_image, float* loss_rows, int B,
                                         int S, int text_rows, int d) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DB200_REQUIRE(B > 0 && S > 0 && text_rows >= 0 && text_rows < S, DB200_E_INVALID,
                "logits_mask_scatter: need B, S > 0 and 0 <= text_rows < S (got B=%d S=%d text_rows=%d)", B, S,
                text_rows);
  DB200_REQUIRE(dx || loss_rows, DB200_E_INVALID, "logits_mask_scatter: nothing to scatter (dx and loss_rows NULL)");
  if (dx) {
    DB200_REQUIRE(d > 0 && d % 8 == 0, DB200_E_INVALID, "logits_mask_scatter: d must be a positive multiple of 8");
    DB200_REQUIRE(dx_image && (text_rows == 0 || dx_text), DB200_E_INVALID, "logits_mask_scatter: NULL dx block");
    DB200_REQUIRE(aligned16(dx) && aligned16(dx_image) && (text_rows == 0 || aligned16(dx_text)), DB200_E_ALIGN,
                  "logits_mask_scatter: dx and its blocks must be 16-byte aligned");
  }
  if (loss_rows)
    DB200_REQUIRE(loss_image && (text_rows == 0 || loss_text), DB200_E_INVALID,
                  "logits_mask_scatter: NULL loss block");
  const long long T = (long long)B * S;
  const int d16 = dx ? d / 8 : 0;
  logits_mask_scatter_kernel<<<grid_for(dx ? T * d16 : T), 256, 0, stream>>>(
      static_cast<const uint4*>(dx_text), static_cast<const uint4*>(dx_image), static_cast<uint4*>(dx), loss_text,
      loss_image, loss_rows, T, S, text_rows, d16);
  return check_launch("logits_mask_scatter_kernel");
}
