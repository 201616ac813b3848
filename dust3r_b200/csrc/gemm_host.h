// Internal host API of the wgmma GEMM (C++ side; the C ABI wrappers live in gemm_host.cu).
#pragma once
#include "gemm_wgmma.cuh"

namespace d3r {
namespace gemm {
// A: [M][lda] bf16 row-major (K valid columns), B: [N][K] bf16.  p.{M,N,K,flags,out,...} filled by the caller.
int gemm_bf16(const void* A, long long lda, const void* B, Params p, cudaStream_t st);
// x: (B,H,W,Cin) bf16 NHWC, w_packed: [Cout][9][Cin] bf16, output (B,H,W,Cout).
int conv3x3_bf16(const void* x_nhwc, const void* w_packed, int B, int H, int W, int Cin, int Cout, Params p, cudaStream_t st);
// k == stride transposed convolution as a GEMM whose epilogue scatters: x (B,h,w,Cin) bf16 NHWC, w_packed
// [(ky*k+kx)*Cout + co][Cin] bf16, bias [Cout] fp32 (may be null), out (B,h*k,w*k,Cout) bf16 NHWC.
int conv_transpose_bf16(const void* x_nhwc, const void* w_packed, void* out, const float* bias, int B, int h, int w, int Cin, int Cout,
                        int k, cudaStream_t st);
// DPT head tail: conv3x3 128->128 (+ bias) -> ReLU -> 1x1 conv to 4 channels (w4 [4][128], b4 [4] fp32) -> pointmap
// postprocess, in the conv's epilogue.  x (B,H,W,128) bf16 NHWC; pts3d (B,H,W,3), conf (B,H,W) fp32 (conf only when
// conf_mode != 0).
int conv3x3_head_tail(const void* x_nhwc, const void* w_packed, const float* bias, const float* w4, const float* b4, float* pts3d,
                      float* conf, int B, int H, int W, int depth_mode, int conf_mode, float conf_min, float conf_max, cudaStream_t st);
}  // namespace gemm
}  // namespace d3r
