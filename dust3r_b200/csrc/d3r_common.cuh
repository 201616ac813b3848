// Shared helpers of the dust3r_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
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

// two floats -> one bf16x2 word (round to nearest even), a in the low half
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 bf16x2_to_float2(uint32_t w) {
  const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&w);
  return make_float2(__low2float(h), __high2float(h));
}

// Pointmap postprocess of pixel `pix` (dust3r/heads/postprocess.py): pts3d = xyz/|xyz| * f(|xyz|), conf = vmin + exp(c)
// (clipped) or a sigmoid.  depth_mode 0 linear, 1 square, 2 exp; conf_mode 0 none, 1 exp, 2 sigmoid.  The confidence
// logit conf_in() is read, and conf written, only when conf_mode != 0.
template <class ConfIn>
__device__ __forceinline__ void postprocess_pixel(float x, float y, float z, ConfIn conf_in, float* pts3d, float* conf, long long pix,
                                                  int depth_mode, int conf_mode, float cmin, float cmax) {
  float ox = x, oy = y, oz = z;
  if (depth_mode != 0) {
    const float d = sqrtf(x * x + y * y + z * z);
    const float dc = fmaxf(d, 1e-8f);
    const float s = (depth_mode == 2) ? expm1f(d) : d * d;
    ox = x / dc * s; oy = y / dc * s; oz = z / dc * s;
  }
  float* o = pts3d + pix * 3;
  o[0] = ox; o[1] = oy; o[2] = oz;
  if (conf_mode != 0) {
    const float c = conf_in();
    float r;
    if (conf_mode == 1) r = cmin + fminf(expf(c), cmax - cmin);
    else r = (cmax - cmin) * (1.f / (1.f + expf(-c))) + cmin;
    conf[pix] = r;
  }
}

int num_sms();

// Tensor map of a bf16 (or `dtype`) tensor for TMA: 128B swizzle, L2 256B promotion, out-of-bounds elements read as zero
// and not written.  dims[0] is the contiguous dimension; strides_bytes holds the rank - 1 outer strides.  `op` names the
// caller in errors.
int encode_tensor_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                      const cuuint32_t* box, const char* op, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);

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
