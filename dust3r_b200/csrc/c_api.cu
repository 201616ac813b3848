// Error reporting + device probing of the dust3r_b200 C ABI, and the host helpers every kernel family shares.
#include "d3r_common.cuh"
#include <cstring>
#include <mutex>

namespace d3r {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode_tensor_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                      const cuuint32_t* box, const char* op, CUtensorMapDataType dtype) {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  if (!fn) {
    set_error("%s: cuTensorMapEncodeTiled is not available from the CUDA driver", op);
    return D3R_ERR_CUDA;
  }
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(m, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("%s: cuTensorMapEncodeTiled failed with CUresult %d (rank %d, dims %llu,%llu)", op, (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1]);
    return D3R_ERR_CUDA;
  }
  return D3R_OK;
}

}  // namespace d3r

extern "C" const char* d3r_last_error(void) { return d3r::g_err; }

extern "C" int d3r_abi_version(void) { return 6; }

extern "C" int d3r_check_device(void) {
  int dev = 0;
  D3R_CUDA(cudaGetDevice(&dev));
  int major = 0, minor = 0;
  D3R_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  D3R_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9 || minor != 0) {
    d3r::set_error("dust3r_b200 is built for sm_90a only; device %d is sm_%d%d", dev, major, minor);
    return D3R_ERR_UNSUPPORTED_DEVICE;
  }
  return D3R_OK;
}
