// Per-thread bodies of the view-stage kernels (csrc/view_ops.cu), written once for device AND host: the kernels call them with
// (blockIdx.x, threadIdx.x), tests/native/view_host.cpp compiles this header with g++ and calls them for every block and thread of
// every launch, so the batching arithmetic, the nearest-neighbour indices and the unprojection are checked bit for bit against
// the reference's numpy / OpenCV code on machines without a GPU.
//
// One launch serves every view of a batch: view v owns blocks [desc[v].blocks[pass], desc[v + 1].blocks[pass]) of the pass; a
// block finds its view by binary search over the descriptors (a few broadcast loads per thread).
//   horizontal pass  image::horizontal_body on the principal-point crop, read in place (src points at its first pixel, the row
//                    pitch is the frame's)
//   vertical pass    image::vertical_pixel, ImgNorm, the store transposed for portrait views
//   depth pass       nearest-neighbour resize + crop, unprojection, camera-to-world transform, valid mask
#pragma once
#include <stdint.h>

#include "../../include/dust3r_b200.h"
#include "hd.h"
#include "resample_core.h"

namespace d3r {
namespace view {

constexpr int kThreads = 256;
enum Pass { kHorizontal = 0, kVertical = 1, kDepth = 2 };

D3R_HD bool finite(float v) { return v == v && v - v == 0.0f; }

// threads of view d in pass p
D3R_HD long long pass_threads(const d3r_view_desc& d, int p) {
  return p == kHorizontal ? (long long)d.rows * d.W2 : (long long)d.H2 * d.W2;
}

// Host side of a call: desc[v].blocks[p] = the first block of view v in pass p, totals[p] = the blocks of pass p.
inline void assign_blocks(d3r_view_desc* desc, int n_views, long long totals[3]) {
  for (int p = 0; p < 3; ++p) totals[p] = 0;
  for (int v = 0; v < n_views; ++v)
    for (int p = 0; p < 3; ++p) {
      desc[v].blocks[p] = totals[p];
      totals[p] += (pass_threads(desc[v], p) + kThreads - 1) / kThreads;
    }
}

// view owning `block` of pass p: the last v with desc[v].blocks[p] <= block
D3R_HD int find_view(const d3r_view_desc* desc, int n_views, long long block, int p) {
  int lo = 0, hi = n_views - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (desc[mid].blocks[p] <= block) lo = mid; else hi = mid - 1;
  }
  return lo;
}

D3R_HD void horizontal_thread(long long block, int thread, const d3r_view_desc* desc, int n_views) {
  const d3r_view_desc& d = desc[find_view(desc, n_views, block, kHorizontal)];
  const image::HorizontalArgs a{d.src, d.src_pitch, d.row0, d.rows, d.crop_x0, d.W2, d.W1, d.xbounds, d.xcoefs, d.tmp};
  image::horizontal_body((block - d.blocks[kHorizontal]) * kThreads + thread, a);
}

D3R_HD void vertical_thread(long long block, int thread, const d3r_view_desc* desc, int n_views, const float* lut) {
  const d3r_view_desc& d = desc[find_view(desc, n_views, block, kVertical)];
  const long long t = (block - d.blocks[kVertical]) * kThreads + thread, plane = (long long)d.H2 * d.W2;
  if (t >= plane) return;
  const int x2 = (int)(t % d.W2), y2 = (int)(t / d.W2);
  const image::VerticalArgs a{d.tmp, d.row0, d.W2, d.H1, d.ybounds, d.ycoefs, d.crop_y0, d.H2, d.W2, lut, nullptr};
  uint8_t rgb[3];
  image::vertical_pixel(a, y2, x2, rgb);
  const long long o = d.transpose ? (long long)x2 * d.H2 + y2 : t;
  d.img[o] = lut[rgb[0]];
  d.img[plane + o] = lut[rgb[1]];
  d.img[2 * plane + o] = lut[rgb[2]];
}

// cv2.resize(INTER_NEAREST) source index of destination index i when n_in samples become n_out
D3R_HD int nearest_index(int i, int n_out, int n_in) {
  const double s = (double)i * (1.0 / ((double)n_out / (double)n_in));
  const int k = (int)s;               // s >= 0: truncation is floor
  return k < n_in - 1 ? k : n_in - 1;
}

D3R_HD void depth_thread(long long block, int thread, const d3r_view_desc* desc, int n_views) {
  const d3r_view_desc& d = desc[find_view(desc, n_views, block, kDepth)];
  const long long t = (block - d.blocks[kDepth]) * kThreads + thread;
  if (t >= (long long)d.H2 * d.W2) return;
  const int x2 = (int)(t % d.W2), y2 = (int)(t / d.W2);
  const int sx = nearest_index(d.crop_x0 + x2, d.W1, d.W0), sy = nearest_index(d.crop_y0 + y2, d.H1, d.H0);
  const float z = d.depth[(long long)sy * d.depth_pitch + sx];
  // the reference's int64 pixel grid promotes the fp32 intrinsics: (u - cu) * z / fu in fp64, rounded once
  const float x = (float)((((double)x2 - (double)d.cu) * (double)z) / (double)d.fu);
  const float y = (float)((((double)y2 - (double)d.cv) * (double)z) / (double)d.fv);
  const float* P = d.pose;
  float w[3];
  for (int i = 0; i < 3; ++i)
    w[i] = fadd(fadd(fadd(fmul(P[4 * i], x), fmul(P[4 * i + 1], y)), fmul(P[4 * i + 2], z)), P[4 * i + 3]);
  const long long o = d.transpose ? (long long)x2 * d.H2 + y2 : t;
  d.depthmap[o] = z;
  d.pts3d[3 * o] = w[0];
  d.pts3d[3 * o + 1] = w[1];
  d.pts3d[3 * o + 2] = w[2];
  d.valid[o] = (uint8_t)(z > 0.0f && finite(w[0]) && finite(w[1]) && finite(w[2]));
}

}  // namespace view
}  // namespace d3r
