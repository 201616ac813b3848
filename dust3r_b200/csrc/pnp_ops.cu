// PnP-RANSAC on the GPU (dust3r_visloc/localization.py: run_pnp, i.e. cv2.solvePnPRansac with SOLVEPNP_SQPNP flags up to its
// final refinement), per-thread bodies in csrc/pnp_core.h.  Hypotheses go in rounds of kRound, every round enqueued up front:
//   pnp_hypothesis_kernel  one thread per hypothesis: its 5-point sample and EPnP in fp64, scratch in shared memory
//   pnp_score_kernel       kHypTile hypotheses' poses in shared memory x kScoreThreads * kPtsPerThread points per block,
//                          per-hypothesis inlier counts in registers, warp-reduced, added to integer counts (order-free)
//   pnp_scan_kernel        one thread: the sequential loop over the round (best, RANSACUpdateNumIters, stop) -> State.done
// and every kernel of a later round returns at once once State.done is set, so no host synchronise sits between rounds.
// pnp_mask_kernel then marks the winning hypothesis' inliers.
#include <algorithm>

#include "d3r_common.cuh"
#include "pnp_core.h"
#include "prof.h"

namespace d3r {
namespace pnp {

constexpr int kRound = 1024;        // hypotheses per round
constexpr int kHypThreads = 32;     // hypotheses (threads) per block of the hypothesis kernel
constexpr int kHypTile = 32;        // hypotheses per block of the scoring kernel
constexpr int kScoreThreads = 256;
constexpr int kPtsPerThread = 4;
constexpr size_t kHypSmem = sizeof(double) * kScratch * kHypThreads;

__device__ __forceinline__ bool round_skipped(const State* st, int32_t h0) { return st && (st->done || h0 >= st->niters); }

__global__ void __launch_bounds__(kHypThreads) pnp_hypothesis_kernel(int32_t n, const float* __restrict__ pts2d,
                                                                     const float* __restrict__ pts3d, Camera cam, uint64_t seed,
                                                                     int32_t h0, int32_t m, const State* st, int32_t* idx_out,
                                                                     double* pose_out, int32_t* counts) {
  if (round_skipped(st, h0)) return;
  extern __shared__ double smem[];
  const int i = blockIdx.x * kHypThreads + threadIdx.x;
  if (i >= m) return;
  const Scratch s{smem + threadIdx.x, kHypThreads};
  int32_t idx[kSample];
  const bool drawn = sample(seed, (uint32_t)(h0 + i), (uint32_t)n, idx);
  bool ok = false;
  if (drawn) {
#pragma unroll
    for (int j = 0; j < kSample; ++j) {
      const long long p = idx[j];
#pragma unroll
      for (int d = 0; d < 3; ++d) s(kPw + 3 * j + d) = (double)pts3d[3 * p + d];
#pragma unroll
      for (int d = 0; d < 2; ++d) s(kUv + 2 * j + d) = (double)pts2d[2 * p + d];
    }
    ok = epnp(s, cam.fx, cam.fy, cam.cx, cam.cy);
  }
#pragma unroll
  for (int j = 0; j < kSample; ++j) idx_out[(long long)kSample * i + j] = drawn ? idx[j] : -1;
#pragma unroll
  for (int k = 0; k < 12; ++k) pose_out[12ll * i + k] = ok ? s(kBest + k) : 0.0;
  counts[i] = ok ? 0 : -1;
}

__global__ void __launch_bounds__(kScoreThreads) pnp_score_kernel(int32_t n, const float* __restrict__ pts2d,
                                                                  const float* __restrict__ pts3d, Camera cam, float thr2,
                                                                  int32_t h0, int32_t m, const State* st,
                                                                  const double* __restrict__ poses, int32_t* counts) {
  if (round_skipped(st, h0)) return;
  __shared__ double pose[kHypTile][12];
  __shared__ int32_t valid[kHypTile], total[kHypTile];
  const int t0 = blockIdx.y * kHypTile;
  for (int k = threadIdx.x; k < kHypTile * 12; k += kScoreThreads) {
    const int hh = k / 12;
    pose[hh][k % 12] = t0 + hh < m ? poses[12ll * (t0 + hh) + k % 12] : 0.0;
  }
  if (threadIdx.x < kHypTile) {
    valid[threadIdx.x] = t0 + (int)threadIdx.x < m && counts[t0 + threadIdx.x] >= 0;
    total[threadIdx.x] = 0;
  }
  __syncthreads();
  float X[kPtsPerThread], Y[kPtsPerThread], Z[kPtsPerThread], u[kPtsPerThread], v[kPtsPerThread];
  bool live[kPtsPerThread];
#pragma unroll
  for (int k = 0; k < kPtsPerThread; ++k) {
    const long long p = ((long long)blockIdx.x * kPtsPerThread + k) * kScoreThreads + threadIdx.x;
    live[k] = p < n;
    const long long q = live[k] ? p : 0;
    X[k] = pts3d[3 * q]; Y[k] = pts3d[3 * q + 1]; Z[k] = pts3d[3 * q + 2];
    u[k] = pts2d[2 * q]; v[k] = pts2d[2 * q + 1];
  }
#pragma unroll 1
  for (int hh = 0; hh < kHypTile; ++hh) {
    if (!valid[hh]) continue;   // uniform across the block
    uint32_t c = 0;
#pragma unroll
    for (int k = 0; k < kPtsPerThread; ++k) c += live[k] && reproj_err2(pose[hh], cam, X[k], Y[k], Z[k], u[k], v[k]) <= thr2;
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&total[hh], (int32_t)c);
  }
  __syncthreads();
  if (threadIdx.x < kHypTile && valid[threadIdx.x] && total[threadIdx.x]) atomicAdd(&counts[t0 + threadIdx.x], total[threadIdx.x]);
}

__global__ void pnp_init_kernel(State* st, int32_t max_iters) { state_init(*st, max_iters); }

__global__ void pnp_scan_kernel(State* st, int32_t h0, int32_t m, const int32_t* counts, const double* poses, int32_t n,
                                double confidence, int32_t* result, double* pose_out) {
  if (st->done) return;
  State s = *st;
  scan_round(s, h0, m, counts, poses, n, confidence);
  *st = s;
  result[0] = s.best;
  result[1] = s.best_count;
  result[2] = s.evaluated;
  result[3] = s.done;
#pragma unroll
  for (int k = 0; k < 12; ++k) pose_out[k] = s.pose[k];
}

__global__ void pnp_mask_kernel(int32_t n, const float* __restrict__ pts2d, const float* __restrict__ pts3d, Camera cam,
                                float thr2, const State* st, uint8_t* mask) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  uint8_t in = 0;
  if (st->best >= 0)
    in = n == kSample || reproj_err2(st->pose, cam, pts3d[3 * p], pts3d[3 * p + 1], pts3d[3 * p + 2], pts2d[2 * p],
                                     pts2d[2 * p + 1]) <= thr2;
  mask[p] = in;
}

static int check_problem(const char* op, int32_t n, const void* pts2d, const void* pts3d, double fx, double fy, double cx,
                         double cy, double threshold) {
  D3R_CHECK_ARG(n >= kSample, "%s: n = %d correspondences, at least %d needed", op, n, kSample);
  D3R_CHECK_ARG(pts2d && pts3d, "%s: null point pointer", op);
  D3R_CHECK_ARG(isfinite(fx) && isfinite(fy) && isfinite(cx) && isfinite(cy) && fx != 0.0 && fy != 0.0,
                "%s: intrinsics (fx %g, fy %g, cx %g, cy %g) must be finite with nonzero focals", op, fx, fy, cx, cy);
  D3R_CHECK_ARG(isfinite(threshold) && threshold >= 0.0, "%s: threshold %g must be finite and >= 0", op, threshold);
  return D3R_OK;
}

static int launch_round(int32_t n, const float* pts2d, const float* pts3d, const Camera& cam, float thr2, uint64_t seed,
                        int32_t h0, int32_t m, const State* st, int32_t* idx, double* poses, int32_t* counts, cudaStream_t stream) {
  // per device, so set on every call (it costs no launch)
  D3R_CUDA(cudaFuncSetAttribute(pnp_hypothesis_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kHypSmem));
  {
    prof::Scope scope("pnp_hypotheses", stream, 0.0, 0.0, 1);
    pnp_hypothesis_kernel<<<(m + kHypThreads - 1) / kHypThreads, kHypThreads, kHypSmem, stream>>>(n, pts2d, pts3d, cam, seed, h0, m,
                                                                                                  st, idx, poses, counts);
    D3R_LAUNCH_CHECK();
  }
  {
    const long long pts_per_block = (long long)kScoreThreads * kPtsPerThread;
    const dim3 grid((unsigned)((n + pts_per_block - 1) / pts_per_block), (unsigned)((m + kHypTile - 1) / kHypTile));
    prof::Scope scope("pnp_score", stream, 30.0 * (double)n * m, 20.0 * (double)n, 1);
    pnp_score_kernel<<<grid, kScoreThreads, 0, stream>>>(n, pts2d, pts3d, cam, thr2, h0, m, st, poses, counts);
    D3R_LAUNCH_CHECK();
  }
  return D3R_OK;
}

}  // namespace pnp
}  // namespace d3r

using namespace d3r;
using namespace d3r::pnp;

extern "C" int64_t d3r_pnp_ransac_workspace_bytes(int32_t max_iters) {
  const int64_t m = std::min<int64_t>(std::max<int32_t>(max_iters, 1), kRound);
  return (int64_t)sizeof(State) + m * (12 * sizeof(double) + (kSample + 1) * sizeof(int32_t));
}

extern "C" int d3r_pnp_hypotheses(int32_t n, const float* pts2d_dev, const float* pts3d_dev, double fx, double fy, double cx,
                                  double cy, double threshold, int64_t seed, int32_t h0, int32_t n_hyp, int32_t* idx_dev,
                                  double* pose_dev, int32_t* counts_dev, void* stream) {
  if (int rc = check_problem("d3r_pnp_hypotheses", n, pts2d_dev, pts3d_dev, fx, fy, cx, cy, threshold)) return rc;
  D3R_CHECK_ARG(h0 >= 0 && n_hyp > 0 && (int64_t)h0 + n_hyp <= INT32_MAX, "d3r_pnp_hypotheses: hypotheses [%d, %d + %d) out of range",
                h0, h0, n_hyp);
  D3R_CHECK_ARG(idx_dev && pose_dev && counts_dev, "d3r_pnp_hypotheses: null output pointer");
  const Camera cam{fx, fy, cx, cy};
  return launch_round(n, pts2d_dev, pts3d_dev, cam, (float)(threshold * threshold), (uint64_t)seed, h0, n_hyp, nullptr, idx_dev,
                      pose_dev, counts_dev, (cudaStream_t)stream);
}

extern "C" int d3r_pnp_ransac(int32_t n, const float* pts2d_dev, const float* pts3d_dev, double fx, double fy, double cx, double cy,
                              double threshold, double confidence, int32_t max_iters, int64_t seed, void* workspace_dev,
                              int64_t workspace_bytes, int32_t* result_dev, double* pose_dev, uint8_t* mask_dev, void* stream) {
  if (int rc = check_problem("d3r_pnp_ransac", n, pts2d_dev, pts3d_dev, fx, fy, cx, cy, threshold)) return rc;
  D3R_CHECK_ARG(confidence > 0.0 && confidence < 1.0, "d3r_pnp_ransac: confidence %g must lie in (0, 1)", confidence);
  D3R_CHECK_ARG(max_iters > 0, "d3r_pnp_ransac: max_iters = %d must be positive", max_iters);
  D3R_CHECK_ARG(workspace_dev && result_dev && pose_dev && mask_dev, "d3r_pnp_ransac: null pointer");
  D3R_CHECK_ARG(workspace_bytes >= d3r_pnp_ransac_workspace_bytes(max_iters), "d3r_pnp_ransac: workspace %lld bytes < %lld needed",
                (long long)workspace_bytes, (long long)d3r_pnp_ransac_workspace_bytes(max_iters));
  D3R_CHECK_ARG(((uintptr_t)workspace_dev & 15) == 0, "d3r_pnp_ransac: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int32_t R = std::min(max_iters, kRound);
  char* ws = (char*)workspace_dev;
  State* state = (State*)ws;
  double* poses = (double*)(ws + sizeof(State));
  int32_t* counts = (int32_t*)(poses + 12ll * R);
  int32_t* idx = counts + R;
  const Camera cam{fx, fy, cx, cy};
  const float thr2 = (float)(threshold * threshold);
  {
    prof::Scope scope("pnp_init", st);
    pnp_init_kernel<<<1, 1, 0, st>>>(state, max_iters);
    D3R_LAUNCH_CHECK();
  }
  for (int32_t h0 = 0; h0 < max_iters; h0 += R) {
    const int32_t m = std::min(R, max_iters - h0);
    if (int rc = launch_round(n, pts2d_dev, pts3d_dev, cam, thr2, (uint64_t)seed, h0, m, state, idx, poses, counts, st)) return rc;
    prof::Scope scope("pnp_scan", st);
    pnp_scan_kernel<<<1, 1, 0, st>>>(state, h0, m, counts, poses, n, confidence, result_dev, pose_dev);
    D3R_LAUNCH_CHECK();
  }
  {
    prof::Scope scope("pnp_mask", st, 0.0, 21.0 * n, 1);
    pnp_mask_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, pts2d_dev, pts3d_dev, cam, thr2, state, mask_dev);
    D3R_LAUNCH_CHECK();
  }
  return D3R_OK;
}
