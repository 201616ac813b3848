// Host harness of the sky segmentation colour test: compiles dust3r_b200/csrc/sky_core.h -- the very per-pixel body the candidate
// kernel of csrc/sky_ops.cu calls -- with g++.  tests/test_sky_host.py runs it over all 2^24 RGB triples and compares H, S, V and
// the candidate bit with cv2.cvtColor(..., COLOR_BGR2HSV) and the reference's thresholds.  Pointers are HOST pointers.
#include "../../dust3r_b200/csrc/sky_core.h"

using namespace d3r::sky;

// rgb [n][3] -> hsv [n][3] (H, S, V as OpenCV's 8-bit HSV), cand [n] (0 / 1)
extern "C" int sky_classify_host(const uint8_t* rgb, long long n, uint8_t* hsv, uint8_t* cand) {
  for (long long i = 0; i < n; ++i) {
    const uint8_t* px = rgb + 3 * i;
    const Hsv p = bgr_to_hsv(px[0], px[1], px[2]);
    hsv[3 * i] = (uint8_t)p.h;
    hsv[3 * i + 1] = (uint8_t)p.s;
    hsv[3 * i + 2] = (uint8_t)p.v;
    cand[i] = sky_candidate(px) ? 1 : 0;
  }
  return 0;
}
