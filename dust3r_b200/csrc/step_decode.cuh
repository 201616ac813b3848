// Device side of the step decoders (JPEG, PNG): one kernel per step of the codec's launch sequence, each running the per-thread
// body Codec::step<S> on one thread per item, and the body of the codec's `d3r_<codec>_decode` / `_workspace_bytes` entry
// points.  The codec's traits struct (Codec in jpeg_core.h / png_core.h) supplies the types, the plan, the launch sequence,
// the Work field that receives the input and the compulsory traffic of one decode.
#pragma once
#include "d3r_common.cuh"
#include "prof.h"

namespace d3r {

constexpr int kStepThreads = 128;

template <class Codec, int S>
__global__ void __launch_bounds__(kStepThreads) step_kernel(int k, typename Codec::Plan P, typename Codec::Work w) {
  Codec::template step<S>((long long)blockIdx.x * blockDim.x + threadIdx.x, k, P, w);
}

// The launcher the codec's `decode` sequence drives on the device; the first error ends the sequence.
template <class Codec>
struct DeviceLauncher {
  cudaStream_t st;
  cudaError_t err = cudaSuccess;
  void zero(void* p, long long bytes) {
    if (err == cudaSuccess) err = cudaMemsetAsync(p, 0, (size_t)bytes, st);
  }
  void copy_desc(void* dst, const typename Codec::Desc* src) {
    if (err == cudaSuccess) err = cudaMemcpyAsync(dst, src, sizeof(typename Codec::Desc), cudaMemcpyHostToDevice, st);
  }
  template <int S>
  void launch(long long n, int k, const typename Codec::Plan& P, const typename Codec::Work& w) {
    if (err != cudaSuccess || n <= 0) return;
    step_kernel<Codec, S><<<(unsigned)((n + kStepThreads - 1) / kStepThreads), kStepThreads, 0, st>>>(k, P, w);
    err = cudaGetLastError();
  }
};

template <class Codec>
int64_t step_decode_workspace_bytes(const typename Codec::Desc* desc, int64_t n_bytes) {
  typename Codec::Plan P;
  if (!desc || Codec::make_plan(*desc, n_bytes, P)) return 0;
  return typename Codec::Layout(P).bytes;
}

template <class Codec>
int step_decode(const typename Codec::Desc* desc, const uint8_t* in_dev, int64_t n_bytes, uint8_t* out_dev, int32_t* status_dev,
                void* workspace_dev, int64_t workspace_bytes, void* stream) {
  const char* name = Codec::kEntry;
  D3R_CHECK_ARG(desc && in_dev && out_dev && status_dev && workspace_dev, "%s: null pointer", name);
  typename Codec::Plan P;
  const char* bad = Codec::make_plan(*desc, n_bytes, P);
  D3R_CHECK_ARG(!bad, "%s: %s", name, bad);
  const typename Codec::Layout lay(P);
  D3R_CHECK_ARG(workspace_bytes >= lay.bytes, "%s: workspace of %lld bytes, need %lld (%s_workspace_bytes)", name,
                (long long)workspace_bytes, lay.bytes, name);
  char* ws = static_cast<char*>(workspace_dev);
  typename Codec::Work w = lay.work(ws);
  w.*Codec::kInput = in_dev;
  w.out = out_dev;
  w.status = status_dev;
  DeviceLauncher<Codec> l{(cudaStream_t)stream};
  {
    prof::Scope scope(Codec::kTag, l.st, 0.0, Codec::traffic(P, n_bytes), Codec::launches(P));
    Codec::decode(l, P, lay, w, *desc, ws);
  }
  if (l.err != cudaSuccess) {
    set_error("%s: %s", name, cudaGetErrorString(l.err));
    return D3R_ERR_CUDA;
  }
  return D3R_OK;
}

}  // namespace d3r
