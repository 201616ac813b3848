// Programmatic dependent launch (PDL) for the forward's kernel chain: every launch carries
// cudaLaunchAttributeProgrammaticStreamSerialization, every kernel does its launch-independent set-up (barrier
// init, tensor-map prefetch) first and then calls pdl::sync_with_predecessor() BEFORE it touches
// any global memory another kernel may have produced or may still be reading.  The next kernel's CTAs are therefore
// scheduled onto SMs as soon as the current kernel's CTAs retire from them, with their prologue already done when the
// predecessor finishes.  A kernel launched without the attribute sees both instructions as no-ops.
// Measured on the 567-launch forward step: no gain (75.5 ms without vs 76.2 ms with, power-capped box) -- the step is
// not launch-gap bound -- so the attribute is OFF by default and D3R_PDL=1 in the environment enables it.  (The
// alignment loop, whose ~10 us serial tail per 77 us iteration does benefit, always uses PDL: align_step.cu.)
#pragma once
#include <cuda_runtime.h>
#include <cstdlib>
#include <utility>

namespace d3r {
namespace pdl {

inline bool enabled() {
  static const bool on = [] {
    const char* e = std::getenv("D3R_PDL");
    return e && e[0] == '1';
  }();
  return on;
}

// wait for the previous grid in the stream to complete and flush, then let the next grid be scheduled (it will
// block at its own wait until THIS grid has completed)
__device__ __forceinline__ void sync_with_predecessor() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// cluster_x > 1: the grid is launched as clusters of cluster_x consecutive CTAs
template <class... KArgs, class... Args>
inline cudaError_t launch_clustered(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster_x,
                                    Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  int n = 0;
  if (enabled()) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster_x > 1) {
    at[n].id = cudaLaunchAttributeClusterDimension;
    at[n].val.clusterDim.x = cluster_x;
    at[n].val.clusterDim.y = 1;
    at[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = at;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

template <class... KArgs, class... Args>
inline cudaError_t launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  return launch_clustered(kernel, grid, block, smem, st, 1, std::forward<Args>(args)...);
}

}  // namespace pdl
}  // namespace d3r
