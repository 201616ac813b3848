// The view stage of evaluation datasets on the GPU (dust3r/datasets/base/base_stereo_view_dataset.py: the principal-point crop,
// the Lanczos / bicubic resize, the nearest-neighbour depth resize, the final crop, ImgNorm, the unprojection to world points
// and the landscape transpose) for a whole batch of RGB-D frames of any mix of sizes: three launches, one per pass, each
// covering every view (csrc/view_core.h).  Byte and fp32 work, HBM-bound: the frames are read once in place (the crop is a
// pointer and a pitch), the intermediate rows of the image resize stay in L2, and each output pixel is written once
// (12 B image, 4 B depth, 12 B points, 1 B mask).
#include <vector>

#include "d3r_common.cuh"
#include "prof.h"
#include "view_core.h"

namespace d3r {
namespace view {

__global__ void __launch_bounds__(kThreads) view_horizontal_kernel(const d3r_view_desc* desc, int n_views) {
  horizontal_thread(blockIdx.x, threadIdx.x, desc, n_views);
}

__global__ void __launch_bounds__(kThreads) view_vertical_kernel(const d3r_view_desc* desc, int n_views, const float* lut) {
  vertical_thread(blockIdx.x, threadIdx.x, desc, n_views, lut);
}

__global__ void __launch_bounds__(kThreads) view_depth_kernel(const d3r_view_desc* desc, int n_views) {
  depth_thread(blockIdx.x, threadIdx.x, desc, n_views);
}

}  // namespace view
}  // namespace d3r

using namespace d3r;
using namespace d3r::view;

extern "C" int32_t d3r_sizeof_view_desc(void) { return (int32_t)sizeof(d3r_view_desc); }

extern "C" int d3r_prepare_views(int32_t n_views, const d3r_view_desc* desc, d3r_view_desc* desc_dev, const float* lut_dev,
                                 void* stream) {
  D3R_CHECK_ARG(n_views > 0, "d3r_prepare_views: n_views = %d must be positive", n_views);
  D3R_CHECK_ARG(desc && desc_dev && lut_dev, "d3r_prepare_views: null pointer");
  std::vector<d3r_view_desc> staged(desc, desc + n_views);
  double src_bytes = 0.0, tmp_px = 0.0, out_px = 0.0;
  for (int v = 0; v < n_views; ++v) {
    const d3r_view_desc& d = staged[v];
    D3R_CHECK_ARG(d.src && d.depth && d.xbounds && d.xcoefs && d.ybounds && d.ycoefs && d.tmp && d.img && d.depthmap && d.pts3d &&
                      d.valid, "d3r_prepare_views: view %d has a null pointer", v);
    D3R_CHECK_ARG(d.H0 > 0 && d.W0 > 0 && d.H1 > 0 && d.W1 > 0 && d.H2 > 0 && d.W2 > 0,
                  "d3r_prepare_views: view %d: sizes must be positive", v);
    D3R_CHECK_ARG(d.src_pitch >= d.W0 && d.depth_pitch >= d.W0, "d3r_prepare_views: view %d: row pitch %d / %d below the width %d", v,
                  d.src_pitch, d.depth_pitch, d.W0);
    D3R_CHECK_ARG(d.crop_x0 >= 0 && d.crop_y0 >= 0 && (long long)d.crop_x0 + d.W2 <= d.W1 && (long long)d.crop_y0 + d.H2 <= d.H1,
                  "d3r_prepare_views: view %d: crop (%d, %d) + %d x %d leaves the resized image %d x %d", v, d.crop_x0, d.crop_y0,
                  d.W2, d.H2, d.W1, d.H1);
    D3R_CHECK_ARG(d.row0 >= 0 && d.rows > 0 && (long long)d.row0 + d.rows <= d.H0,
                  "d3r_prepare_views: view %d: source rows [%d, %d) outside [0, %d)", v, d.row0, d.row0 + d.rows, d.H0);
    src_bytes += 3.0 * d.rows * d.W0 + 4.0 * d.H2 * d.W2;
    tmp_px += (double)d.rows * d.W2;
    out_px += (double)d.H2 * d.W2;
  }
  long long blocks[3];
  assign_blocks(staged.data(), n_views, blocks);
  for (int p = 0; p < 3; ++p)
    D3R_CHECK_ARG(blocks[p] < (1ll << 31), "d3r_prepare_views: batch too large (%lld blocks in one launch)", blocks[p]);
  cudaStream_t st = (cudaStream_t)stream;
  // pageable source: the copy has left `staged` when cudaMemcpyAsync returns
  D3R_CUDA(cudaMemcpyAsync(desc_dev, staged.data(), sizeof(d3r_view_desc) * n_views, cudaMemcpyHostToDevice, st));
  {
    prof::Scope scope("view_resample_h", st, 0.0, src_bytes + 3.0 * tmp_px, 1);
    view_horizontal_kernel<<<(unsigned)blocks[kHorizontal], kThreads, 0, st>>>(desc_dev, n_views);
    D3R_LAUNCH_CHECK();
  }
  {
    prof::Scope scope("view_resample_v", st, 0.0, 3.0 * tmp_px + 12.0 * out_px, 1);
    view_vertical_kernel<<<(unsigned)blocks[kVertical], kThreads, 0, st>>>(desc_dev, n_views, lut_dev);
    D3R_LAUNCH_CHECK();
  }
  {
    prof::Scope scope("view_depth", st, 0.0, 21.0 * out_px, 1);
    view_depth_kernel<<<(unsigned)blocks[kDepth], kThreads, 0, st>>>(desc_dev, n_views);
    D3R_LAUNCH_CHECK();
  }
  return D3R_OK;
}
