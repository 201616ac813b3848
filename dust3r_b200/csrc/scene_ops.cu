// Scene-level kernels either side of the alignment loop (SURVEY §8f "next" rows), sm_90a:
//   * clean_pointcloud          cross-view consistency filter                 dust3r/cloud_opt/base_opt.py:369-405
//   * weighted Procrustes sums  moments of weighted Umeyama / Kabsch          roma.rigid_points_registration as called by
//                                                                             dust3r/cloud_opt/init_im_poses.py:66-110, 253-262
//   * Weiszfeld focal           IRLS focal from a pointmap                    dust3r/post_process.py:12-60
//   * nearest neighbours        brute-force 3-D NN for reciprocal matching    dust3r/utils/geometry.py:345-361 (cKDTree there)
// All are HBM / L2 streaming reductions or maps over pixels: one thread per pixel, coalesced fp32 loads, warp-shuffle + block
// reductions, fp64 accumulation where sums are later differenced (Procrustes moments).  The 3x3 SVD, clipping and graph logic stay
// on the host side (dust3r_b200/cloud_opt/scene_ops.py).
#include "d3r_common.cuh"
#include "prof.h"

namespace d3r {
namespace scene {

constexpr int kThreads = 256;

// ------------------------------------------------------------------------------------------------ clean_pointcloud
// Image i, pixel p: its world point X is expressed in every other camera j, rounded to the pixel it lands on, and if it lies
// in front of j's surface there ((1 - tol) * depth_j) while j is the more confident of the two, conf_i[p] is cut to bad_conf.
// The reference visits (i, j) sequentially and later tests see the confidences lowered by earlier ones: one launch per image
// i (in order), one thread per pixel walking j = 0..n-1 -- conf of images < i is final, of images > i untouched, and pixel p
// of image i only depends on itself.
__global__ void __launch_bounds__(kThreads) clean_kernel(int i, int n, const int* __restrict__ hw, const long long* __restrict__ off,
                                                         const float* __restrict__ pts, float* conf, const float* __restrict__ depth,
                                                         const float* __restrict__ Kmat, const float* __restrict__ cams, float tol,
                                                         float bad_conf) {
  const int P = hw[2 * i] * hw[2 * i + 1];
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const long long o = off[i] + p;
  const float x = pts[3 * o], y = pts[3 * o + 1], z = pts[3 * o + 2];
  float c = conf[o];
  for (int j = 0; j < n; ++j) {
    if (j == i) continue;
    const float* T = cams + 16 * j;     // world -> camera j, row-major 4x4 (geotrf: R X + t)
    const float px = T[0] * x + T[1] * y + T[2] * z + T[3];
    const float py = T[4] * x + T[5] * y + T[6] * z + T[7];
    const float pz = T[8] * x + T[9] * y + T[10] * z + T[11];
    const float* Kj = Kmat + 9 * j;     // geotrf(K, proj, norm=1, ncol=2): (K proj)[:2] / (K proj)[2]
    const float qx = Kj[0] * px + Kj[1] * py + Kj[2] * pz;
    const float qy = Kj[3] * px + Kj[4] * py + Kj[5] * pz;
    const float qz = Kj[6] * px + Kj[7] * py + Kj[8] * pz;
    const float uf = rintf(qx / qz), vf = rintf(qy / qz);     // torch.round: half to even
    const int Hj = hw[2 * j], Wj = hw[2 * j + 1];
    if (!(pz > 0.f) || !(uf >= 0.f) || !(uf < float(Wj)) || !(vf >= 0.f) || !(vf < float(Hj))) continue;
    const long long q = off[j] + (long long)vf * Wj + (long long)uf;
    if (pz < (1.f - tol) * depth[q] && c < conf[q]) c = fminf(c, bad_conf);
  }
  conf[o] = c;
}

// ------------------------------------------------------------------------------------------------ Procrustes moments
// Per problem b: sum w, sum w x (3), sum w y (3), sum w y x^T (9), sum w |x|^2 -> 17 doubles.  grid = (chunks, B).
constexpr int kMom = 17;
__global__ void __launch_bounds__(kThreads) procrustes_kernel(int P, const float* __restrict__ x, const float* __restrict__ y,
                                                              const float* __restrict__ w, double* __restrict__ out) {
  const int b = blockIdx.y;
  const float* xb = x + (long long)b * P * 3;
  const float* yb = y + (long long)b * P * 3;
  const float* wb = w + (long long)b * P;
  double m[kMom];
#pragma unroll
  for (int k = 0; k < kMom; ++k) m[k] = 0.0;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < P; p += gridDim.x * blockDim.x) {
    const float ww = wb[p];
    const float x0 = xb[3 * p], x1 = xb[3 * p + 1], x2 = xb[3 * p + 2];
    const float y0 = yb[3 * p], y1 = yb[3 * p + 1], y2 = yb[3 * p + 2];
    const double wd = ww;
    m[0] += wd;
    m[1] += wd * x0; m[2] += wd * x1; m[3] += wd * x2;
    m[4] += wd * y0; m[5] += wd * y1; m[6] += wd * y2;
    m[7] += wd * y0 * x0; m[8] += wd * y0 * x1; m[9] += wd * y0 * x2;
    m[10] += wd * y1 * x0; m[11] += wd * y1 * x1; m[12] += wd * y1 * x2;
    m[13] += wd * y2 * x0; m[14] += wd * y2 * x1; m[15] += wd * y2 * x2;
    m[16] += wd * (double(x0) * x0 + double(x1) * x1 + double(x2) * x2);
  }
  __shared__ double s[kThreads / 32][kMom];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kMom; ++k) {
    double v = m[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) s[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < kMom) {
    double v = 0.0;
#pragma unroll
    for (int ww = 0; ww < kThreads / 32; ++ww) v += s[ww][threadIdx.x];
    atomicAdd(out + (long long)b * kMom + threadIdx.x, v);
  }
}

// ------------------------------------------------------------------------------------------------ Weiszfeld focal
// One CTA per pointmap.  rays = (x/z, y/z) (non-finite -> 0), num = <ray, px>, den = <ray, ray>;
// f0 = mean(num) / mean(den); 10 x: w = 1 / max(|px - f ray|, 1e-8); f = mean(w num) / mean(w den).  (post_process.py:36-58)
__device__ __forceinline__ float finite_or_zero(float v) { return (fabsf(v) <= 3.4028234e38f) ? v : 0.f; }   // NaN -> 0 too

__global__ void __launch_bounds__(1024) weiszfeld_kernel(int H, int W, const float* __restrict__ pts, const float* __restrict__ pp,
                                                          int steps, float* __restrict__ out) {
  const int b = blockIdx.x;
  const int P = H * W;
  const float* pb = pts + (long long)b * P * 3;
  const float cx = pp[2 * b], cy = pp[2 * b + 1];
  __shared__ double s_a[32], s_b[32];
  __shared__ float s_focal;
  float focal = 0.f;
  for (int it = 0; it <= steps; ++it) {
    double a = 0.0, d = 0.0;
    for (int p = threadIdx.x; p < P; p += blockDim.x) {
      const float x = pb[3 * p], y = pb[3 * p + 1], z = pb[3 * p + 2];
      const float rx = finite_or_zero(x / z), ry = finite_or_zero(y / z);   // nan_to_num(posinf=0, neginf=0) maps NaN to 0 as well
      const int v = p / W, u = p - v * W;
      const float ux = float(u) - cx, uy = float(v) - cy;
      const float num = rx * ux + ry * uy, den = rx * rx + ry * ry;
      float wgt = 1.f;
      if (it > 0) {
        const float ex = ux - focal * rx, ey = uy - focal * ry;
        wgt = 1.f / fmaxf(sqrtf(ex * ex + ey * ey), 1e-8f);
      }
      a += double(wgt * num);
      d += double(wgt * den);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); d += __shfl_xor_sync(0xffffffffu, d, o); }
    if (lane == 0) { s_a[warp] = a; s_b[warp] = d; }
    __syncthreads();
    if (threadIdx.x == 0) {
      double ta = 0.0, tb = 0.0;
      for (int k = 0; k < int(blockDim.x >> 5); ++k) { ta += s_a[k]; tb += s_b[k]; }
      s_focal = float(ta / tb);
    }
    __syncthreads();
    focal = s_focal;
    __syncthreads();
  }
  if (threadIdx.x == 0) out[b] = focal;
}

// ------------------------------------------------------------------------------------------------ nearest neighbours
// For every query a_i the index of the closest point of B (squared Euclidean distance, lowest index on ties): B is streamed
// through shared memory in tiles, one thread per query.
constexpr int kTile = 2048;
__global__ void __launch_bounds__(kThreads) nn_kernel(int N, int M, const float* __restrict__ A, const float* __restrict__ B,
                                                      int* __restrict__ nn) {
  __shared__ float4 tile[kTile];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float ax = 0.f, ay = 0.f, az = 0.f;
  if (i < N) { ax = A[3 * i]; ay = A[3 * i + 1]; az = A[3 * i + 2]; }
  float best = INFINITY;
  int arg = 0;
  for (int t0 = 0; t0 < M; t0 += kTile) {
    const int cnt = min(kTile, M - t0);
    __syncthreads();
    for (int k = threadIdx.x; k < cnt; k += blockDim.x) tile[k] = make_float4(B[3 * (t0 + k)], B[3 * (t0 + k) + 1], B[3 * (t0 + k) + 2], 0.f);
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < cnt; ++k) {
      const float4 q = tile[k];
      const float dx = ax - q.x, dy = ay - q.y, dz = az - q.z;
      const float d2 = fmaf(dx, dx, fmaf(dy, dy, dz * dz));
      if (d2 < best) { best = d2; arg = t0 + k; }
    }
  }
  if (i < N) nn[i] = arg;
}

}  // namespace scene
}  // namespace d3r

using namespace d3r;
using namespace d3r::scene;

extern "C" int d3r_clean_pointcloud(int32_t n_imgs, const int32_t* hw_dev, const int64_t* off_dev, int32_t max_area, const float* pts3d_dev,
                                    float* conf_dev, const float* depth_dev, const float* K_dev, const float* cams_dev, float tol,
                                    float bad_conf, void* stream) {
  D3R_CHECK_ARG(n_imgs > 0 && hw_dev && off_dev && pts3d_dev && conf_dev && depth_dev && K_dev && cams_dev && max_area > 0,
                "d3r_clean_pointcloud: bad arguments");
  D3R_CHECK_ARG(tol >= 0.f && tol < 1.f, "d3r_clean_pointcloud: tol must be in [0, 1)");
  prof::Scope scope("clean_pointcloud", (cudaStream_t)stream, 0.0, 0.0, n_imgs);
  const int blocks = (max_area + kThreads - 1) / kThreads;
  for (int i = 0; i < n_imgs; ++i)
    clean_kernel<<<blocks, kThreads, 0, (cudaStream_t)stream>>>(i, n_imgs, hw_dev, reinterpret_cast<const long long*>(off_dev), pts3d_dev,
                                                              conf_dev, depth_dev, K_dev, cams_dev, tol, bad_conf);
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}

extern "C" int d3r_procrustes_moments(int32_t n_problems, int32_t n_points, const float* x_dev, const float* y_dev, const float* w_dev,
                                      double* out_dev, void* stream) {
  D3R_CHECK_ARG(n_problems > 0 && n_points > 0 && x_dev && y_dev && w_dev && out_dev, "d3r_procrustes_moments: bad arguments");
  D3R_CHECK_ARG(n_problems <= 65535, "d3r_procrustes_moments: too many problems (%d) for one launch", n_problems);
  D3R_CUDA(cudaMemsetAsync(out_dev, 0, sizeof(double) * kMom * size_t(n_problems), (cudaStream_t)stream));
  int bx = (n_points + kThreads * 8 - 1) / (kThreads * 8);
  if (bx > 64) bx = 64;
  prof::Scope scope("procrustes_moments", (cudaStream_t)stream, 0.0, double(n_problems) * n_points * 28.0, 1);
  procrustes_kernel<<<dim3((unsigned)bx, (unsigned)n_problems), kThreads, 0, (cudaStream_t)stream>>>(n_points, x_dev, y_dev, w_dev, out_dev);
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}

extern "C" int d3r_weiszfeld_focal(int32_t n_maps, int32_t H, int32_t W, const float* pts3d_dev, const float* pp_dev, int32_t steps,
                                   float* focal_dev, void* stream) {
  D3R_CHECK_ARG(n_maps > 0 && H > 0 && W > 0 && pts3d_dev && pp_dev && focal_dev && steps >= 0, "d3r_weiszfeld_focal: bad arguments");
  prof::Scope scope("weiszfeld_focal", (cudaStream_t)stream, 0.0, double(n_maps) * H * W * 12.0 * (steps + 1), 1);
  weiszfeld_kernel<<<n_maps, 1024, 0, (cudaStream_t)stream>>>(H, W, pts3d_dev, pp_dev, steps, focal_dev);
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}

extern "C" int d3r_nearest_neighbours(int32_t n_queries, int32_t n_points, const float* queries_dev, const float* points_dev,
                                      int32_t* nn_dev, void* stream) {
  D3R_CHECK_ARG(n_queries > 0 && n_points > 0 && queries_dev && points_dev && nn_dev, "d3r_nearest_neighbours: bad arguments");
  prof::Scope scope("nearest_neighbours", (cudaStream_t)stream, 8.0 * double(n_queries) * n_points, 0.0, 1);
  nn_kernel<<<(n_queries + kThreads - 1) / kThreads, kThreads, 0, (cudaStream_t)stream>>>(n_queries, n_points, queries_dev, points_dev, nn_dev);
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}
