// Shared helpers of the dust3r_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>

#include "../../include/dust3r_b200.h"

namespace d3r {

void set_error(const char* fmt, ...);

#define D3R_CHECK_ARG(cond, ...)                    \
  do {                                              \
    if (!(cond)) {                                  \
      ::d3r::set_error(__VA_ARGS__);                \
      return D3R_ERR_INVALID;                       \
    }                                               \
  } while (0)

#define D3R_CUDA(expr)                                                                     \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      ::d3r::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return D3R_ERR_CUDA;                                                                 \
    }                                                                                      \
  } while (0)

#define D3R_LAUNCH_CHECK()                                                                 \
  do {                                                                                     \
    cudaError_t _e = cudaGetLastError();                                                   \
    if (_e != cudaSuccess) {                                                               \
      ::d3r::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return D3R_ERR_CUDA;                                                                 \
    }                                                                                      \
  } while (0)

__device__ __forceinline__ float warp_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v;
}

int num_sms();

// cudaFuncSetAttribute is per device / context: a launch site keeps one bit per device in a static mask and opts in the first time it
// launches on each device of the process (a process may drive several GPUs: global_aligner(out, 'cuda:1') next to a model on cuda:0)
inline bool first_launch_on_this_device(unsigned long long& mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (mask & bit) return false;
  mask |= bit;
  return true;
}

}  // namespace d3r
