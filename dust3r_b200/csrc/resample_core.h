// Per-thread bodies of the image preprocessing kernels (csrc/image_ops.cu), written once for device AND host: the CUDA kernels
// call them with t = blockIdx.x * blockDim.x + threadIdx.x, tests/native/resample_host.cpp compiles this very header with g++ and
// calls them in a loop over t, so the index arithmetic and the integer resampling that run on the GPU are checked bit for bit
// against Pillow on machines without a GPU.
//
// What is computed (dust3r/utils/image.py:62-71 `_resize_pil_image`, :101-124 crop + ImgNorm, i.e. Pillow's Image.resize for
// 8-bit images = two separable passes of src/libImaging/Resample.c, Image.crop, torchvision ToTensor + Normalize(0.5, 0.5)):
//   horizontal pass   tmp[y][x][c] = clip8((2^21 + sum_i src[y][lo_x + i][c] * kx[x][i]) >> 22)      uint8 -> uint8
//   vertical pass     out[c][y][x] = lut[clip8((2^21 + sum_i tmp[lo_y + i][x][c] * ky[y][i]) >> 22)]   uint8 -> fp32 CHW
// (one thread per PIXEL, three accumulators) with 22-bit fixed-point coefficient tables, stored tap-major, built on the host (dust3r_b200/utils/image.py: Pillow's precompute_coeffs /
// normalize_coeffs_8bpc in double precision) and lut[v] = (v / 255 - 0.5) / 0.5 as torch computes it on the CPU.  Only the
// rows / columns of the intermediate image that the cropped output reads are produced.
#pragma once
#include <stdint.h>

#include "hd.h"

namespace d3r {
namespace image {

constexpr int kPrecisionBits = 22;   // Resample.c PRECISION_BITS = 32 - 8 - 2

// Resample.c clip8: arithmetic shift, then clamp to [0, 255]
D3R_HD uint8_t clip8(uint32_t acc) {
  const int32_t v = (int32_t)acc >> kPrecisionBits;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

struct HorizontalArgs {
  const uint8_t* src;      // [H0][W0][3] decoded RGB
  int32_t W0;              // source row length in pixels
  int32_t row0, rows;      // source rows the vertical pass will read: [row0, row0 + rows)
  int32_t col0, cols;      // resized columns that survive the crop: [col0, col0 + cols)
  int32_t W1;              // resized row length = row pitch of the tap-major coefficient table
  const int32_t* bounds;   // [W1][2] first source column, tap count
  const int32_t* coefs;    // [ksize][W1] tap-major: neighbouring threads (columns) read neighbouring coefficients
  uint8_t* tmp;            // [rows][cols][3]
};

// thread t -> pixel (row yi, column xi) of tmp, all three channels (one coefficient load serves R, G and B); xi fastest, so a
// warp reads one contiguous stretch of a source row per tap and writes 96 contiguous bytes
D3R_HD void horizontal_body(long long t, const HorizontalArgs& a) {
  const long long total = (long long)a.rows * a.cols;
  if (t >= total) return;
  const int xi = (int)(t % a.cols);
  const int yi = (int)(t / a.cols);
  const int x = a.col0 + xi;
  const int lo = a.bounds[2 * x], cnt = a.bounds[2 * x + 1];
  const int32_t* k = a.coefs + x;
  const uint8_t* p = a.src + ((long long)(a.row0 + yi) * a.W0 + lo) * 3;
  uint32_t r = 1u << (kPrecisionBits - 1), g = r, b = r;
  for (int i = 0; i < cnt; ++i) {
    const int32_t w = k[(long long)i * a.W1];
    r += (uint32_t)((int32_t)p[3 * i] * w);
    g += (uint32_t)((int32_t)p[3 * i + 1] * w);
    b += (uint32_t)((int32_t)p[3 * i + 2] * w);
  }
  uint8_t* q = a.tmp + t * 3;
  q[0] = clip8(r);
  q[1] = clip8(g);
  q[2] = clip8(b);
}

struct VerticalArgs {
  const uint8_t* tmp;      // [rows][cols][3] written by the horizontal pass
  int32_t row0, cols;      // as above
  int32_t H1;              // resized height = row pitch of the tap-major coefficient table
  const int32_t* bounds;   // [H1][2] first source row, tap count
  const int32_t* coefs;    // [ksize][H1] tap-major
  int32_t crop_y0;         // first resized row of the crop
  int32_t H2, W2;          // output size (W2 == cols)
  const float* lut;        // [256]
  float* out;              // [3][H2][W2]
};

// The resampled bytes of output pixel (y2, x2), before ImgNorm: the vertical pass of every caller (vertical_body below and the
// view stage of view_core.h, which stores them elsewhere).  `out` is not read.
D3R_HD void vertical_pixel(const VerticalArgs& a, int y2, int x2, uint8_t rgb[3]) {
  const int y1 = a.crop_y0 + y2;
  const int lo = a.bounds[2 * y1] - a.row0, cnt = a.bounds[2 * y1 + 1];
  const int32_t* k = a.coefs + y1;
  const long long pitch = (long long)a.cols * 3;
  const uint8_t* p = a.tmp + (long long)lo * pitch + (long long)x2 * 3;
  uint32_t r = 1u << (kPrecisionBits - 1), g = r, b = r;
  for (int i = 0; i < cnt; ++i) {
    const int32_t w = k[(long long)i * a.H1];
    const uint8_t* q = p + i * pitch;
    r += (uint32_t)((int32_t)q[0] * w);
    g += (uint32_t)((int32_t)q[1] * w);
    b += (uint32_t)((int32_t)q[2] * w);
  }
  rgb[0] = clip8(r);
  rgb[1] = clip8(g);
  rgb[2] = clip8(b);
}

// thread t -> pixel (row y2, column x2) of out, all three channel planes; x2 fastest: a warp reads 96 contiguous bytes of an
// intermediate row per tap (the coefficient is the same for the whole row: a broadcast load) and writes three coalesced
// 128-byte lines
D3R_HD void vertical_body(long long t, const VerticalArgs& a) {
  const long long plane = (long long)a.H2 * a.W2;
  if (t >= plane) return;
  uint8_t rgb[3];
  vertical_pixel(a, (int)(t / a.W2), (int)(t % a.W2), rgb);
  a.out[t] = a.lut[rgb[0]];
  a.out[plane + t] = a.lut[rgb[1]];
  a.out[2 * plane + t] = a.lut[rgb[2]];
}

}  // namespace image
}  // namespace d3r
