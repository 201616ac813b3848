// Sky segmentation on the GPU (BasePCOptimizer.mask_sky, dust3r/cloud_opt/base_opt.py:289-295, built on dust3r/viz.py:345-381
// `segment_sky`), bit-exact, for n images of any mix of sizes in one call:
//   1. candidate   OpenCV's 8-bit HSV of the RGB bytes read as BGR + the reference's thresholds (sky_core.h)
//   2. erosion     5x5, zero padding: a pixel survives when its whole window is a candidate (so nothing within 2 of the border does)
//   3. dilation    5x5, zero padding: foreground = any eroded pixel in the window  (2 + 3 = scipy.ndimage.binary_opening)
//   4. labelling   8-connected components by lock-free union-find over global pixel indices (so no union crosses images): every
//                  foreground pixel unites with its foreground W / NW / N / NE neighbours, roots are linked to the smaller index
//                  by CAS (Playne & Hawick 2018 / ECL-CC style, intermediate pointer jumping while merging), then every
//                  label is replaced by its root
//   5. areas       integer atomics per root (warp-aggregated: the pixels of one row of a component share a root), per-image max
//   6. select      sky = foreground && 2 * area[root] > max area of the image   (the reference's "area > max / 2" set)
// Seven launches whatever the content: the union-find needs no host loop that iterates until labels converge.  The result is a
// set, not a labelling, so it is deterministic although the labels the atomics produce are not.
// Memory: the candidate mask is staged in the output buffer; the workspace holds the eroded mask, the labels, the areas and the
// per-image maxima (d3r_segment_sky_workspace_bytes).
#include "d3r_common.cuh"
#include "prof.h"
#include "sky_core.h"

namespace d3r {
namespace sky {

constexpr int kThreads = 256;
constexpr int kRadius = 2;   // 5x5 structuring element

struct Images {
  const int* hw;            // [n][2]
  const long long* off;     // [n] first pixel of image i
};

// blockIdx.y = image, blockIdx.x * blockDim.x + threadIdx.x = pixel of that image; false past its end
struct Pixel {
  long long g;   // global pixel index
  int y, x, H, W;
};

__device__ __forceinline__ bool locate(const Images& im, Pixel& p) {
  const int i = blockIdx.y;
  p.H = im.hw[2 * i];
  p.W = im.hw[2 * i + 1];
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= p.H * p.W) return false;
  p.y = q / p.W;
  p.x = q - p.y * p.W;
  p.g = im.off[i] + q;
  return true;
}

__global__ void __launch_bounds__(kThreads) candidate_kernel(Images im, const uint8_t* __restrict__ rgb, uint8_t* __restrict__ cand) {
  Pixel p;
  if (!locate(im, p)) return;
  cand[p.g] = sky_candidate(rgb + 3 * p.g) ? 1 : 0;
}

// every pixel of the 5x5 window is a candidate (all false within kRadius of the border: the padding is 0)
__global__ void __launch_bounds__(kThreads) erode_kernel(Images im, const uint8_t* __restrict__ cand, uint8_t* __restrict__ ero) {
  Pixel p;
  if (!locate(im, p)) return;
  bool keep = p.y >= kRadius && p.y < p.H - kRadius && p.x >= kRadius && p.x < p.W - kRadius;
  for (int dy = -kRadius; keep && dy <= kRadius; ++dy) {
    const uint8_t* row = cand + p.g + (long long)dy * p.W;
#pragma unroll
    for (int dx = -kRadius; dx <= kRadius; ++dx) keep = keep && row[dx];
  }
  ero[p.g] = keep ? 1 : 0;
}

// foreground = any eroded pixel in the 5x5 window (clipped to the image); initialises the union-find (label = own index for the
// foreground, -1 for the background), zeroes the areas and the image's maximum
__global__ void __launch_bounds__(kThreads) dilate_init_kernel(Images im, const uint8_t* __restrict__ ero, int* __restrict__ label,
                                                               int* __restrict__ area, int* __restrict__ max_area) {
  if (blockIdx.x == 0 && threadIdx.x == 0) max_area[blockIdx.y] = 0;
  Pixel p;
  if (!locate(im, p)) return;
  const int y0 = max(p.y - kRadius, 0), y1 = min(p.y + kRadius, p.H - 1);
  const int x0 = max(p.x - kRadius, 0) - p.x, x1 = min(p.x + kRadius, p.W - 1) - p.x;
  bool fg = false;
  for (int y = y0; !fg && y <= y1; ++y) {
    const uint8_t* row = ero + p.g + (long long)(y - p.y) * p.W;
    for (int dx = x0; dx <= x1; ++dx) fg = fg || row[dx];
  }
  label[p.g] = fg ? (int)p.g : -1;
  area[p.g] = 0;
}

// root of x: follows parent links (always to a smaller index).  While roots are still being linked (the merge kernel) every
// visited node is pointed at its grandparent on the way; afterwards the walk is read-only, so that the roots the flatten kernel
// stores are never overwritten by another thread's shortcut.  The loads bypass L1: other SMs relink roots concurrently and a
// stale L1 line would only cost extra rounds.
template <bool kCompress>
__device__ __forceinline__ int find_root(int* label, int x) {
  int cur = __ldcg(label + x);
  if (cur != x) {
    int prev = x, next;
    while (cur > (next = __ldcg(label + cur))) {
      if (kCompress) label[prev] = next;
      prev = cur;
      cur = next;
    }
  }
  return cur;
}

// links the roots of a and b, the larger index below the smaller; a failed CAS means that root was linked meanwhile: retry from
// its new parent
__device__ __forceinline__ void unite(int* label, int a, int b) {
  int ra = find_root<true>(label, a), rb = find_root<true>(label, b);
  while (ra != rb) {
    if (ra < rb) {
      const int old = atomicCAS(label + rb, rb, ra);
      if (old == rb) break;
      rb = old;
    } else {
      const int old = atomicCAS(label + ra, ra, rb);
      if (old == ra) break;
      ra = old;
    }
  }
}

// 8-connectivity with four unions at most, usually one: a foreground N neighbour is already connected to NW, W and NE (they are
// its own W, SW and E neighbours), and a foreground W to NW (its N)
__global__ void __launch_bounds__(kThreads) merge_kernel(Images im, int* label) {
  Pixel p;
  if (!locate(im, p)) return;
  const int g = (int)p.g;
  if (__ldcg(label + g) < 0) return;
  const bool up = p.y > 0, left = p.x > 0, right = p.x + 1 < p.W;
  const int n = g - p.W;
  if (up && __ldcg(label + n) >= 0) {
    unite(label, g, n);
    return;
  }
  if (left && __ldcg(label + g - 1) >= 0) unite(label, g, g - 1);
  else if (up && left && __ldcg(label + n - 1) >= 0) unite(label, g, n - 1);
  if (up && right && __ldcg(label + n + 1) >= 0) unite(label, g, n + 1);
}

// label = root; area[root] += 1, one atomic per distinct root of the warp
__global__ void __launch_bounds__(kThreads) flatten_count_kernel(Images im, int* label, int* __restrict__ area) {
  Pixel p;
  int root = -1;
  if (locate(im, p)) {
    root = __ldcg(label + p.g);
    if (root >= 0) {
      root = find_root<false>(label, (int)p.g);
      label[p.g] = root;
    }
  }
  const unsigned peers = __match_any_sync(0xffffffffu, root);
  if (root >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(area + root, __popc(peers));
}

__global__ void __launch_bounds__(kThreads) max_area_kernel(Images im, const int* __restrict__ label, const int* __restrict__ area,
                                                            int* __restrict__ max_area) {
  Pixel p;
  if (!locate(im, p)) return;
  if (label[p.g] == (int)p.g) atomicMax(max_area + blockIdx.y, area[p.g]);
}

__global__ void __launch_bounds__(kThreads) select_kernel(Images im, const int* __restrict__ label, const int* __restrict__ area,
                                                          const int* __restrict__ max_area, uint8_t* __restrict__ out) {
  Pixel p;
  if (!locate(im, p)) return;
  const int root = label[p.g];
  out[p.g] = (root >= 0 && 2ll * area[root] > (long long)max_area[blockIdx.y]) ? 1 : 0;
}

// compulsory DRAM / L2 traffic per pixel, windows and union chains served by L1 / L2 counted once: candidate 3 + 1, erode 1 + 1,
// dilate_init 1 + 4 + 4, merge 4, flatten_count 4 + 4, max_area 4 + 4, select 4 + 4 + 1
constexpr double kBytesPerPixel = 44.0;

constexpr long long kAlign = 256;
__host__ __forceinline__ long long align_up(long long b) { return (b + kAlign - 1) / kAlign * kAlign; }

// [labels int32 x total][areas int32 x total][maxima int32 x n][eroded uint8 x total], each 256-byte aligned
struct Layout {
  long long label, area, max_area, ero, bytes;
  Layout(int n, long long total) {
    label = 0;
    area = label + align_up(4 * total);
    max_area = area + align_up(4 * total);
    ero = max_area + align_up(4ll * n);
    bytes = ero + align_up(total);
  }
};

}  // namespace sky
}  // namespace d3r

using namespace d3r;
using namespace d3r::sky;

extern "C" int64_t d3r_segment_sky_workspace_bytes(int32_t n_imgs, int64_t total_px) {
  if (n_imgs <= 0 || total_px <= 0) return 0;
  return Layout(n_imgs, total_px).bytes;
}

extern "C" int d3r_segment_sky(int32_t n_imgs, const int32_t* hw_dev, const int64_t* off_dev, int32_t max_area, int64_t total_px,
                               const uint8_t* rgb_dev, uint8_t* sky_out_dev, void* workspace_dev, int64_t workspace_bytes, void* stream) {
  D3R_CHECK_ARG(hw_dev && off_dev && rgb_dev && sky_out_dev && workspace_dev, "d3r_segment_sky: null pointer");
  D3R_CHECK_ARG(n_imgs > 0 && n_imgs <= 65535, "d3r_segment_sky: n_imgs = %d outside [1, 65535]", n_imgs);
  D3R_CHECK_ARG(max_area > 0 && total_px >= max_area && total_px <= (long long)n_imgs * max_area,
                "d3r_segment_sky: total_px = %lld inconsistent with %d images of at most %d pixels", (long long)total_px, n_imgs, max_area);
  // labels are global pixel indices in int32
  D3R_CHECK_ARG(total_px < (1ll << 31), "d3r_segment_sky: %lld pixels exceed the 2^31-pixel label range", (long long)total_px);
  const Layout lay(n_imgs, total_px);
  D3R_CHECK_ARG(workspace_bytes >= lay.bytes, "d3r_segment_sky: workspace of %lld bytes, need %lld (d3r_segment_sky_workspace_bytes)",
                (long long)workspace_bytes, lay.bytes);
  char* ws = static_cast<char*>(workspace_dev);
  int* label = reinterpret_cast<int*>(ws + lay.label);
  int* area = reinterpret_cast<int*>(ws + lay.area);
  int* maxa = reinterpret_cast<int*>(ws + lay.max_area);
  uint8_t* ero = reinterpret_cast<uint8_t*>(ws + lay.ero);
  const Images im{hw_dev, reinterpret_cast<const long long*>(off_dev)};
  const dim3 grid((unsigned)((max_area + kThreads - 1) / kThreads), (unsigned)n_imgs);
  cudaStream_t st = (cudaStream_t)stream;
  prof::Scope scope("segment_sky", st, 0.0, double(total_px) * kBytesPerPixel, 7);
  candidate_kernel<<<grid, kThreads, 0, st>>>(im, rgb_dev, sky_out_dev);
  erode_kernel<<<grid, kThreads, 0, st>>>(im, sky_out_dev, ero);
  dilate_init_kernel<<<grid, kThreads, 0, st>>>(im, ero, label, area, maxa);
  merge_kernel<<<grid, kThreads, 0, st>>>(im, label);
  flatten_count_kernel<<<grid, kThreads, 0, st>>>(im, label, area);
  max_area_kernel<<<grid, kThreads, 0, st>>>(im, label, area, maxa);
  select_kernel<<<grid, kThreads, 0, st>>>(im, label, area, maxa, sky_out_dev);
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}
