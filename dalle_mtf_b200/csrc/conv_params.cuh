// Parameter blocks shared by the CUDA-core (conv.cu) and tensor-core fp32 (conv_f32_tc.cu) convolution kernels.
#pragma once
#include "common.cuh"

namespace db200 {

constexpr int MAX_TAPS = 16;

struct Tap {
  int dy, dx;       // source pixel = (oy*in_stride + dy, ox*in_stride + dx)
  long long w_off;  // element offset of this tap's [K][N] slab in the weight tensor
};

struct ConvGemmParams {
  int NB, OH, OW;          // enumeration grid of output pixels (M = NB*OH*OW)
  int out_H, out_W;        // spatial dims of the output tensor
  int out_stride, oa, ob;  // output pixel = (oy*out_stride + oa, ox*out_stride + ob)
  int in_H, in_W, in_stride;
  int K, Nn;               // channels contracted / produced
  int ntaps;
  Tap taps[MAX_TAPS];
  long long w_k_stride, w_n_stride;
  const void* x;
  const float* w;
  const float* bias;
  const void* residual;  // same layout/dtype as y
  const void* mask;      // same layout/dtype as y: y *= (mask > 0)
  void* y;
  int relu;
};

struct WgradTap {
  int pdy, pdx, qdy, qdx;
  long long w_off;
};
struct ConvWgradParams {
  int NB, OH, OW;  // enumeration grid (contracted)
  int pH, pW, pC, p_stride;
  int qH, qW, qC, q_stride;
  int ntaps, splits;
  WgradTap taps[MAX_TAPS];
  long long a_stride, b_stride;
  const void* P;
  const void* Q;
  float* dw;
};


// conv_f32_tc.cu: fp32 activations on wgmma through a three-way bf16 split (fp32-accurate products)
bool conv_gemm_f32_tc_ok(const ConvGemmParams& p);
int conv_gemm_f32_tc_launch(cudaStream_t stream, const ConvGemmParams& p);
bool conv_wgrad_f32_tc_ok(const ConvWgradParams& p);
int conv_wgrad_f32_tc_launch(cudaStream_t stream, ConvWgradParams& p);

}  // namespace db200
