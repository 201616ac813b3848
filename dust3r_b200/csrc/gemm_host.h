// Internal host API of the wgmma GEMM (C++ side; the C ABI wrappers live in gemm_host.cu).
#pragma once
#include "gemm_wgmma.cuh"

namespace d3r {
namespace gemm {
// A: [M][lda] bf16 row-major (K valid columns), B: [N][K] bf16.  p.{M,N,K,flags,out,...} filled by the caller.
int gemm_bf16(const void* A, long long lda, const void* B, Params p, cudaStream_t st);
// x: (B,H,W,Cin) bf16 NHWC, w_packed: [Cout][9][Cin] bf16, output (B,H,W,Cout).
int conv3x3_bf16(const void* x_nhwc, const void* w_packed, int B, int H, int W, int Cin, int Cout, Params p, cudaStream_t st);
}  // namespace gemm
}  // namespace d3r
