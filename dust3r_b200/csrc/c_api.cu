// Error reporting + device probing of the dust3r_b200 C ABI.
#include "d3r_common.cuh"
#include <cstring>

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

}  // namespace d3r

extern "C" const char* d3r_last_error(void) { return d3r::g_err; }

extern "C" int d3r_abi_version(void) { return 3; }

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
