// Host harness of the PnP-RANSAC kernels: compiles dust3r_b200/csrc/pnp_core.h -- the very per-thread bodies of csrc/pnp_ops.cu --
// with g++ (-ffp-contract=off).  tests/test_pnp_host.py runs every thread index of small launches against oracle/pnp_float64.py.
// Pointers are HOST pointers; layouts are those of d3r_pnp_hypotheses / d3r_pnp_ransac.
#include <vector>

#include "../../dust3r_b200/csrc/pnp_core.h"

using namespace d3r::pnp;

// hypotheses h0 .. h0 + m - 1: the body of pnp_hypothesis_kernel (thread i) and of pnp_score_kernel (its counts)
extern "C" int pnp_hypotheses_host(int32_t n, const float* pts2d, const float* pts3d, double fx, double fy, double cx, double cy,
                                   double threshold, uint64_t seed, int32_t h0, int32_t m, int32_t* idx_out, double* pose_out,
                                   int32_t* counts) {
  std::vector<double> scratch(kScratch);
  const Scratch s{scratch.data(), 1};
  const Camera cam{fx, fy, cx, cy};
  const float thr2 = (float)(threshold * threshold);
  for (int32_t i = 0; i < m; ++i) {
    int32_t idx[kSample];
    const bool drawn = sample(seed, (uint32_t)(h0 + i), (uint32_t)n, idx);
    bool ok = false;
    if (drawn) {
      for (int j = 0; j < kSample; ++j) {
        for (int d = 0; d < 3; ++d) s(kPw + 3 * j + d) = (double)pts3d[3 * (long long)idx[j] + d];
        for (int d = 0; d < 2; ++d) s(kUv + 2 * j + d) = (double)pts2d[2 * (long long)idx[j] + d];
      }
      ok = epnp(s, fx, fy, cx, cy);
    }
    for (int j = 0; j < kSample; ++j) idx_out[kSample * i + j] = drawn ? idx[j] : -1;
    for (int k = 0; k < 12; ++k) pose_out[12 * i + k] = ok ? s(kBest + k) : 0.0;
    int32_t c = -1;
    if (ok) {
      c = 0;
      for (int32_t p = 0; p < n; ++p)
        c += reproj_err2(pose_out + 12 * i, cam, pts3d[3 * p], pts3d[3 * p + 1], pts3d[3 * p + 2], pts2d[2 * p], pts2d[2 * p + 1]) <= thr2;
    }
    counts[i] = c;
  }
  return 0;
}

// EPnP of one 5-point sample given as fp64 arrays (pw [5][3], uv [5][2]); returns 1 and Rt when valid
extern "C" int pnp_epnp_host(const double* pw, const double* uv, double fx, double fy, double cx, double cy, double* Rt) {
  std::vector<double> scratch(kScratch);
  const Scratch s{scratch.data(), 1};
  for (int k = 0; k < 15; ++k) s(kPw + k) = pw[k];
  for (int k = 0; k < 10; ++k) s(kUv + k) = uv[k];
  if (!epnp(s, fx, fy, cx, cy)) return 0;
  for (int k = 0; k < 12; ++k) Rt[k] = s(kBest + k);
  return 1;
}

extern "C" int pnp_err2_host(const double* Rt, double fx, double fy, double cx, double cy, int32_t n, const float* pts2d,
                             const float* pts3d, float* err) {
  const Camera cam{fx, fy, cx, cy};
  for (int32_t p = 0; p < n; ++p)
    err[p] = reproj_err2(Rt, cam, pts3d[3 * p], pts3d[3 * p + 1], pts3d[3 * p + 2], pts2d[2 * p], pts2d[2 * p + 1]);
  return 0;
}

extern "C" int pnp_update_num_iters_host(double p, double ep, int32_t model_points, int32_t max_iters) {
  return update_num_iters(p, ep, model_points, max_iters);
}

// the whole loop in rounds of `round` hypotheses, as d3r_pnp_ransac runs it: result {best, count, evaluated, done}
extern "C" int pnp_ransac_host(int32_t n, const float* pts2d, const float* pts3d, double fx, double fy, double cx, double cy,
                               double threshold, double confidence, int32_t max_iters, uint64_t seed, int32_t round,
                               int32_t* result, double* pose, uint8_t* mask) {
  State st;
  state_init(st, max_iters);
  std::vector<int32_t> idx(kSample * round), counts(round);
  std::vector<double> poses(12 * round);
  for (int32_t h0 = 0; h0 < max_iters && !st.done; h0 += round) {
    const int32_t m = round < max_iters - h0 ? round : max_iters - h0;
    if (h0 >= st.niters) break;
    pnp_hypotheses_host(n, pts2d, pts3d, fx, fy, cx, cy, threshold, seed, h0, m, idx.data(), poses.data(), counts.data());
    scan_round(st, h0, m, counts.data(), poses.data(), n, confidence);
  }
  result[0] = st.best;
  result[1] = st.best_count;
  result[2] = st.evaluated;
  result[3] = st.done;
  for (int k = 0; k < 12; ++k) pose[k] = st.pose[k];
  const Camera cam{fx, fy, cx, cy};
  const float thr2 = (float)(threshold * threshold);
  for (int32_t p = 0; p < n; ++p)
    mask[p] = st.best >= 0 && (n == kSample || reproj_err2(st.pose, cam, pts3d[3 * p], pts3d[3 * p + 1], pts3d[3 * p + 2],
                                                           pts2d[2 * p], pts2d[2 * p + 1]) <= thr2);
  return 0;
}
