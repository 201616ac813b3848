// Host harness of the view-stage kernels: compiles dust3r_b200/csrc/view_core.h -- the very per-thread bodies the CUDA kernels
// of csrc/view_ops.cu call -- with g++ and runs them for every block and thread of the three launches d3r_prepare_views makes
// (block assignment included, so the ragged last block of every view runs too).  tests/test_views_host.py compares the result
// with the reference's Pillow / OpenCV / numpy view stage bit for bit, on machines without a GPU.  The descriptors hold HOST
// pointers here.
#include "../../dust3r_b200/csrc/view_core.h"

using namespace d3r::view;

extern "C" int view_host(int32_t n_views, d3r_view_desc* desc, const float* lut) {
  long long blocks[3];
  assign_blocks(desc, n_views, blocks);
  for (long long b = 0; b < blocks[kHorizontal]; ++b)
    for (int t = 0; t < kThreads; ++t) horizontal_thread(b, t, desc, n_views);
  for (long long b = 0; b < blocks[kVertical]; ++b)
    for (int t = 0; t < kThreads; ++t) vertical_thread(b, t, desc, n_views, lut);
  for (long long b = 0; b < blocks[kDepth]; ++b)
    for (int t = 0; t < kThreads; ++t) depth_thread(b, t, desc, n_views);
  return 0;
}
