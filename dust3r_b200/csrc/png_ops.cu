// PNG decode on the GPU, bit-identical to Pillow: the per-thread bodies and the launch sequence are in png_core.h (shared with
// the host harness tests/native/png_host.cpp); this file turns each step into a kernel.  Every step is one thread per item
// (stream byte, subsequence, block, inflated byte, Adler segment, row); the kernels differ only in the body they run.
#include "d3r_common.cuh"
#include "png_core.h"
#include "prof.h"

namespace d3r {
namespace png {

constexpr int kThreads = 128;

template <int S>
__global__ void __launch_bounds__(kThreads) png_step_kernel(int k, Plan P, Work w) {
  step<S>((long long)blockIdx.x * blockDim.x + threadIdx.x, k, P, w);
}

struct DeviceLauncher {
  cudaStream_t st;
  cudaError_t err = cudaSuccess;
  void zero(void* p, long long bytes) {
    if (err == cudaSuccess) err = cudaMemsetAsync(p, 0, (size_t)bytes, st);
  }
  void copy_desc(void* dst, const d3r_png_desc* src) {
    if (err == cudaSuccess) err = cudaMemcpyAsync(dst, src, sizeof(d3r_png_desc), cudaMemcpyHostToDevice, st);
  }
  template <int S>
  void launch(long long n, int k, const Plan& P, const Work& w) {
    if (err != cudaSuccess || n <= 0) return;
    png_step_kernel<S><<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, st>>>(k, P, w);
    err = cudaGetLastError();
  }
};

}  // namespace png
}  // namespace d3r

using namespace d3r;
using namespace d3r::png;

extern "C" int32_t d3r_sizeof_png_desc(void) { return (int32_t)sizeof(d3r_png_desc); }

extern "C" int64_t d3r_png_decode_workspace_bytes(const d3r_png_desc* desc, int64_t n_bytes) {
  Plan P;
  if (!desc || make_plan(*desc, n_bytes, P)) return 0;
  return Layout(P).bytes;
}

extern "C" int d3r_png_decode(const d3r_png_desc* desc, const uint8_t* zdata_dev, int64_t n_bytes, uint8_t* out_dev,
                              int32_t* status_dev, void* workspace_dev, int64_t workspace_bytes, void* stream) {
  D3R_CHECK_ARG(desc && zdata_dev && out_dev && status_dev && workspace_dev, "d3r_png_decode: null pointer");
  Plan P;
  const char* bad = make_plan(*desc, n_bytes, P);
  D3R_CHECK_ARG(!bad, "d3r_png_decode: %s", bad);
  const Layout lay(P);
  D3R_CHECK_ARG(workspace_bytes >= lay.bytes, "d3r_png_decode: workspace of %lld bytes, need %lld (d3r_png_decode_workspace_bytes)",
                (long long)workspace_bytes, lay.bytes);
  char* ws = static_cast<char*>(workspace_dev);
  Work w = lay.work(ws);
  w.z = zdata_dev;
  w.out = out_dev;
  w.status = status_dev;
  DeviceLauncher l{(cudaStream_t)stream};
  {
    // compulsory traffic: the stream (read about three times), the inflated rows and their roots written, read and written
    // again, the RGB out
    const double bytes = 3.0 * double(n_bytes) + 4.0 * double(P.total) + 8.0 * double(P.total) + 3.0 * double(P.W) * P.H;
    prof::Scope scope("png_decode", l.st, 0.0, bytes, P.rounds + 8);
    decode(l, P, lay, w, *desc, ws);
  }
  if (l.err != cudaSuccess) {
    set_error("d3r_png_decode: %s", cudaGetErrorString(l.err));
    return D3R_ERR_CUDA;
  }
  return D3R_OK;
}
