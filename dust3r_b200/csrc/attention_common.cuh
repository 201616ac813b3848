// Helpers of the attention kernels (attention_wgmma.cu).
#pragma once
#include "d3r_common.cuh"
#include "sm90_ptx.cuh"
#include <mutex>

namespace d3r {
namespace attn {
namespace tcc {

__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static inline EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// tokens of one image: [N][ld] bf16 -> 3-D map {cols, N, B}, box {64, box_rows, 1}: rows past N are zero-filled
static inline int make_map(CUtensorMap* m, const void* base, long long ld, int cols, int N, int B, int box_rows) {
  EncodeTiledFn fn = get_encode();
  if (!fn) { set_error("cuTensorMapEncodeTiled unavailable"); return D3R_ERR_CUDA; }
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)N, (cuuint64_t)B};
  cuuint64_t str[2] = {(cuuint64_t)ld * 2, (cuuint64_t)N * ld * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, str, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("attention: cuTensorMapEncodeTiled failed (%d)", (int)r); return D3R_ERR_CUDA; }
  return D3R_OK;
}


}  // namespace tcc
}  // namespace attn
}  // namespace d3r
