// Qualifiers and explicitly rounded arithmetic for the per-thread bodies in the *_core.h headers, which nvcc compiles into the
// kernels and g++ compiles into the host harnesses of tests/native.
//   D3R_HD           a body both sides run, inlined on the device
//   D3R_HD_NOINLINE  a body the device calls as a function of its own (a separate register allocation)
//   D3R_UNROLL       #pragma unroll for nvcc, nothing for g++ (which would warn about an unknown pragma)
//   D3R_UNROLL_BY(n) #pragma unroll n, likewise
#pragma once

#if defined(__CUDACC__)
#define D3R_HD __host__ __device__ __forceinline__
#define D3R_HD_NOINLINE __host__ __device__ __noinline__
#define D3R_PRAGMA(text) _Pragma(#text)
#define D3R_UNROLL D3R_PRAGMA(unroll)
#define D3R_UNROLL_BY(n) D3R_PRAGMA(unroll n)
#else
#define D3R_HD inline
#define D3R_HD_NOINLINE inline
#define D3R_UNROLL
#define D3R_UNROLL_BY(n)
#endif

namespace d3r {

// Each operation rounded on its own: nvcc would contract a multiply and an add into an FMA, numpy and OpenCV do not (the host
// harnesses are built with -ffp-contract=off).  In namespace d3r because glibc declares C23 fadd / fmul / fsub globally.
#if defined(__CUDA_ARCH__)
D3R_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
D3R_HD double dadd(double a, double b) { return __dadd_rn(a, b); }
D3R_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
D3R_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
D3R_HD float fsub(float a, float b) { return __fsub_rn(a, b); }
#else
D3R_HD double dmul(double a, double b) { return a * b; }
D3R_HD double dadd(double a, double b) { return a + b; }
D3R_HD float fmul(float a, float b) { return a * b; }
D3R_HD float fadd(float a, float b) { return a + b; }
D3R_HD float fsub(float a, float b) { return a - b; }
#endif

}  // namespace d3r
