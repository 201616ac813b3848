// Per-pixel body of the sky segmentation kernels (csrc/sky_ops.cu), written once for device AND host: the candidate kernel calls
// it for every pixel, tests/native/sky_host.cpp compiles this very header with g++ and runs it over all 2^24 RGB triples, so the
// colour test the GPU executes is checked bit for bit against OpenCV on machines without a GPU.
//
// What is computed (dust3r/viz.py:345-381 `segment_sky`, colour part):
//   hsv = cv2.cvtColor(q, COLOR_BGR2HSV) on an RGB array, i.e. channel 0 plays "blue" and channel 2 plays "red".  This is OpenCV's
//   8-bit HSV (modules/imgproc/src/color_hsv: 12-bit fixed-point reciprocal tables, H in [0, 180)):
//     v = max, diff = max - min, s = (diff * round(255 * 2^12 / v) + 2^11) >> 12   (0 when v == 0)
//     h = c1 - c0 (v == c2), else c0 - c2 + 2 diff (v == c1), else c2 - c1 + 4 diff;
//     h = (h * round(180 * 2^12 / (6 diff)) + 2^11) >> 12 (0 when diff == 0), + 180 when negative
//   (neither reciprocal ever lands on a half, so the rounding mode of OpenCV's table build does not matter);
//   candidate = (H <= 30 & V >= 100) | (S < 10 & V > 150) | (S < 30 & V > 180) | (S < 50 & V > 220).
#pragma once
#include <stdint.h>

#include "hd.h"

namespace d3r {
namespace sky {

constexpr int kHsvShift = 12;

struct Hsv {
  int32_t h, s, v;
};

// c0, c1, c2 = the three bytes of one pixel in memory order (R, G, B of the scene images)
D3R_HD Hsv bgr_to_hsv(int32_t c0, int32_t c1, int32_t c2) {
  int32_t v = c0 > c1 ? c0 : c1;
  v = v > c2 ? v : c2;
  int32_t mn = c0 < c1 ? c0 : c1;
  mn = mn < c2 ? mn : c2;
  const int32_t diff = v - mn;
  const int32_t sdiv = v ? (2 * (255 << kHsvShift) + v) / (2 * v) : 0;                    // round(255 * 2^12 / v)
  const int32_t hdiv = diff ? (2 * (180 << kHsvShift) + 6 * diff) / (12 * diff) : 0;     // round(180 * 2^12 / (6 diff))
  const int32_t s = (diff * sdiv + (1 << (kHsvShift - 1))) >> kHsvShift;
  int32_t h = v == c2 ? c1 - c0 : (v == c1 ? c0 - c2 + 2 * diff : c2 - c1 + 4 * diff);
  h = (h * hdiv + (1 << (kHsvShift - 1))) >> kHsvShift;
  h += h < 0 ? 180 : 0;
  return Hsv{h, s, v};
}

// inRange(hsv, (0, 0, 100), (30, 255, 255)) plus the three "luminous gray" terms
D3R_HD bool sky_candidate(const Hsv& p) {
  return (p.h <= 30 && p.v >= 100) || (p.s < 10 && p.v > 150) || (p.s < 30 && p.v > 180) || (p.s < 50 && p.v > 220);
}

D3R_HD bool sky_candidate(const uint8_t* px) { return sky_candidate(bgr_to_hsv(px[0], px[1], px[2])); }

}  // namespace sky
}  // namespace d3r
