// Per-thread bodies of the PnP-RANSAC kernels (csrc/pnp_ops.cu), written once for device AND host: the kernels call them, and
// tests/native/pnp_host.cpp compiles this very header with g++ so the sample draws, the EPnP solver, the inlier test and the
// stopping rule are checked against oracle/pnp_float64.py on machines without a GPU.
//
// What is computed: OpenCV's solvePnPRansac loop with SOLVEPNP_SQPNP flags (calib3d/src/solvepnp.cpp and ptsetreg.cpp), whose
// minimal solver is EPnP on 5-point samples, with one deliberate difference, the random draws:
//
//   * Samples.  Hypothesis h draws indices from a stateless counter-based generator, SplitMix64's finaliser:
//       z(h, k) = mix64(seed + 0x9E3779B97F4A7C15 * ((h << 32 | k) + 1))          (uint64 arithmetic, wrapping)
//       draw k  = (z >> 32) * n >> 32                                             (an index in [0, n))
//     for k = 0, 1, 2, ...; a draw equal to one already taken is rejected, until 5 distinct indices are held, in draw order.
//     After kMaxDraws draws without 5 distinct indices the hypothesis is invalid (never for n >= 6 in practice).  With n == 5
//     the only sample is {0, 1, 2, 3, 4}, and the loop is OpenCV's "count == modelPoints" branch: one EPnP on all points, no
//     scoring, every point an inlier.
//   * Minimal solver.  EPnP (Lepetit, Moreno-Noguer & Fua, 2009) in fp64, as OpenCV's calib3d/src/epnp.cpp: PCA control
//     points, barycentric coordinates, the 12x12 M^T M and its four eigenvectors of smallest eigenvalue (cyclic Jacobi), the
//     beta estimates for N = 1, 2, 3 each refined by 5 Gauss-Newton steps, and the solution of least mean reprojection error.
//     Four choices OpenCV leaves to its SVD: the sign of each PCA direction (its component of largest magnitude is made
//     positive; the control points, and so the pose from noisy points, depend on it); a PCA direction whose eigenvalue is below kFlat times the largest is flat (its
//     control point is the centroid and its barycentric coordinate 0: the pseudo-inverse of the control-point matrix); the
//     two eigenvectors of smallest eigenvalue span the exact null space of the 10 x 12 M, in which an eigensolver picks an
//     arbitrary basis, so they are replaced by a canonical one (v[0] along the projection of kCanon onto that plane, v[1]
//     orthogonal to it), which makes the pose a function of the sample alone; and the rotation of each solution is the
//     proper rotation closest to the camera/world cross-covariance (Horn's quaternion method, equal to U V^T whenever
//     det(U V^T) > 0).  A sample with a non-finite result is invalid: 0 inliers, never NaN.
//   * Scoring (PnPRansacCallback::computeError + RANSACPointSetRegistrator::findInliers): points as fp32, the projection
//     x = R X + t in fp64 in projectPoints' operation order, z -> 1/z (1 when z == 0), u = x fx + cx rounded to fp32, the
//     squared error in fp32 and inlier when err <= fp32(thr^2).  No cheirality test.  Every operation is explicitly rounded
//     (no FMA contraction), so host and device give the same bits.
//   * Stopping rule (RANSACPointSetRegistrator::run): hypotheses in index order; one becomes the best when its count is
//     > max(best count, 4), and then niters = RANSACUpdateNumIters(confidence, (n - count) / n, 5, niters).  The loop ends
//     after hypothesis niters - 1.
#pragma once
#include <math.h>
#include <stdint.h>

#include "hd.h"

namespace d3r {
namespace pnp {

constexpr int kSample = 5;           // points per EPnP sample (OpenCV's model_points for every flag but P3P / AP3P)
constexpr int kMaxDraws = 1024;      // draws per hypothesis before it is invalid
constexpr int kJacobiSweeps = 30;    // cap on cyclic Jacobi sweeps (12x12 converges in < 10)
constexpr int kGaussNewton = 5;      // Gauss-Newton steps per beta estimate (epnp.cpp: gauss_newton)
constexpr double kFlat = 1e-30;      // PCA eigenvalue ratio below which a direction is flat (OpenCV inverts all but exact 0)
constexpr uint64_t kDefaultSeed = 0x5DEECE66Dull;

// ---- sample draws ----
D3R_HD uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

D3R_HD uint32_t draw(uint64_t seed, uint32_t h, uint32_t k, uint32_t n) {
  const uint64_t z = mix64(seed + 0x9E3779B97F4A7C15ull * ((((uint64_t)h) << 32 | k) + 1ull));
  return (uint32_t)(((z >> 32) * (uint64_t)n) >> 32);
}

// the 5 indices of hypothesis h (draw order); false when kMaxDraws draws did not give 5 distinct ones
D3R_HD bool sample(uint64_t seed, uint32_t h, uint32_t n, int32_t idx[kSample]) {
  if (n == (uint32_t)kSample) {
D3R_UNROLL
    for (int j = 0; j < kSample; ++j) idx[j] = j;
    return true;
  }
  int m = 0;
  for (uint32_t k = 0; k < (uint32_t)kMaxDraws && m < kSample; ++k) {
    const int32_t i = (int32_t)draw(seed, h, k, n);
    bool dup = false;
D3R_UNROLL
    for (int j = 0; j < kSample; ++j) dup |= (j < m) && idx[j] == i;
    if (!dup) {
D3R_UNROLL
      for (int j = 0; j < kSample; ++j)
        if (j == m) idx[j] = i;
      ++m;
    }
  }
  return m == kSample;
}

// ---- EPnP scratch: kScratch doubles per thread, element k at p[k * stride] (stride = threads of the block on the device,
// so the threads of a warp touch consecutive words; 1 on the host) ----
struct Scratch {
  double* p;
  int stride;
  D3R_HD double& operator()(int k) const { return p[(long long)k * stride]; }
};

enum : int {
  kA = 0,                  // 12x12 symmetric matrix being diagonalised (also the 3x3 / 4x4 ones)
  kV = kA + 144,           // its eigenvectors (columns)
  kPw = kV + 144,          // [5][3] world points
  kUv = kPw + 15,          // [5][2] pixels
  kAlpha = kUv + 10,       // [5][4] barycentric coordinates
  kCw = kAlpha + 20,       // [4][3] world control points
  kNull = kCw + 12,        // [4][12] null-space vectors, v[0] of the smallest eigenvalue
  kL = kNull + 48,         // [6][10]
  kRho = kL + 60,          // [6]
  kQ = kRho + 6,           // [6][5] least-squares matrix
  kRhs = kQ + 30,          // [6]
  kDiag = kRhs + 6,        // [5]
  kX = kDiag + 5,          // [5] least-squares solution
  kBeta = kX + 5,          // [4]
  kCc = kBeta + 4,         // [4][3] camera control points
  kPc = kCc + 12,          // [5][3] camera points
  kRt = kPc + 15,          // [12] candidate R (row-major) | t
  kBest = kRt + 12,        // [12] best solution so far
  kScratch = kBest + 12
};

// The EPnP stages below are D3R_HD_NOINLINE: separate register allocations, no spills.

// cyclic Jacobi on the n x n symmetric matrix at s(kA): eigenvalues on its diagonal, eigenvectors in the columns of s(kV).
// Rotations as in Numerical Recipes' jacobi: after 4 sweeps an element negligible against both diagonal entries is set to
// 0; the loop ends when every off-diagonal element is 0 (or a NaN appeared).
D3R_HD_NOINLINE void jacobi(Scratch s, int n) {
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) s(kV + i * n + j) = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < n; ++p)
      for (int q = p + 1; q < n; ++q) off += fabs(s(kA + p * n + q));
    if (!(off > 0.0)) break;
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        const double apq = s(kA + p * n + q);
        const double app = s(kA + p * n + p), aqq = s(kA + q * n + q);
        const double g = 100.0 * fabs(apq);
        if (sweep > 3 && fabs(app) + g == fabs(app) && fabs(aqq) + g == fabs(aqq)) {
          s(kA + p * n + q) = 0.0;
          s(kA + q * n + p) = 0.0;
          continue;
        }
        if (apq == 0.0) continue;
        const double theta = (aqq - app) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
        for (int k = 0; k < n; ++k) {
          if (k == p || k == q) continue;
          const double akp = s(kA + k * n + p), akq = s(kA + k * n + q);
          const double np = c * akp - sn * akq, nq = sn * akp + c * akq;
          s(kA + k * n + p) = np;
          s(kA + p * n + k) = np;
          s(kA + k * n + q) = nq;
          s(kA + q * n + k) = nq;
        }
        s(kA + p * n + p) = app - t * apq;
        s(kA + q * n + q) = aqq + t * apq;
        s(kA + p * n + q) = 0.0;
        s(kA + q * n + p) = 0.0;
        for (int k = 0; k < n; ++k) {
          const double vkp = s(kV + k * n + p), vkq = s(kV + k * n + q);
          s(kV + k * n + p) = c * vkp - sn * vkq;
          s(kV + k * n + q) = sn * vkp + c * vkq;
        }
      }
  }
}

// least squares min |Q x - rhs| for the 6 x ncol matrix at s(kQ) (row stride 5) by Householder QR; x at s(kX).  False when a
// column is (numerically) dependent on the previous ones.
D3R_HD_NOINLINE bool lsq6(Scratch s, int ncol) {
  for (int k = 0; k < ncol; ++k) {
    double nrm = 0.0;
    for (int i = k; i < 6; ++i) nrm += s(kQ + i * 5 + k) * s(kQ + i * 5 + k);
    nrm = sqrt(nrm);
    if (!(nrm > 0.0)) return false;
    const double alpha = s(kQ + k * 5 + k) > 0.0 ? -nrm : nrm;
    s(kQ + k * 5 + k) -= alpha;
    double vtv = 0.0;
    for (int i = k; i < 6; ++i) vtv += s(kQ + i * 5 + k) * s(kQ + i * 5 + k);
    if (!(vtv > 0.0)) return false;
    for (int j = k + 1; j < ncol; ++j) {
      double d = 0.0;
      for (int i = k; i < 6; ++i) d += s(kQ + i * 5 + k) * s(kQ + i * 5 + j);
      const double f = 2.0 * d / vtv;
      for (int i = k; i < 6; ++i) s(kQ + i * 5 + j) -= f * s(kQ + i * 5 + k);
    }
    double d = 0.0;
    for (int i = k; i < 6; ++i) d += s(kQ + i * 5 + k) * s(kRhs + i);
    const double f = 2.0 * d / vtv;
    for (int i = k; i < 6; ++i) s(kRhs + i) -= f * s(kQ + i * 5 + k);
    s(kDiag + k) = alpha;
  }
  for (int j = ncol - 1; j >= 0; --j) {
    double r = s(kRhs + j);
    for (int l = j + 1; l < ncol; ++l) r -= s(kQ + j * 5 + l) * s(kX + l);
    s(kX + j) = r / s(kDiag + j);
  }
  return true;
}

// the pairs of control points, in epnp.cpp's order
D3R_HD void pair_of(int k, int& a, int& b) {
  a = k < 3 ? 0 : (k < 5 ? 1 : 2);
  b = k < 3 ? k + 1 : (k < 5 ? k - 1 : 3);
}

// Gauss-Newton on the 6 distance equations from the betas at s(kBeta) (epnp.cpp: compute_A_and_b_gauss_newton, qr_solve)
D3R_HD_NOINLINE void gauss_newton(Scratch s) {
  for (int it = 0; it < kGaussNewton; ++it) {
    const double b0 = s(kBeta), b1 = s(kBeta + 1), b2 = s(kBeta + 2), b3 = s(kBeta + 3);
    for (int i = 0; i < 6; ++i) {
      const int r = kL + 10 * i;
      s(kQ + i * 5 + 0) = 2 * s(r) * b0 + s(r + 1) * b1 + s(r + 3) * b2 + s(r + 6) * b3;
      s(kQ + i * 5 + 1) = s(r + 1) * b0 + 2 * s(r + 2) * b1 + s(r + 4) * b2 + s(r + 7) * b3;
      s(kQ + i * 5 + 2) = s(r + 3) * b0 + s(r + 4) * b1 + 2 * s(r + 5) * b2 + s(r + 8) * b3;
      s(kQ + i * 5 + 3) = s(r + 6) * b0 + s(r + 7) * b1 + s(r + 8) * b2 + 2 * s(r + 9) * b3;
      s(kRhs + i) = s(kRho + i) - (s(r) * b0 * b0 + s(r + 1) * b0 * b1 + s(r + 2) * b1 * b1 + s(r + 3) * b0 * b2 +
                                   s(r + 4) * b1 * b2 + s(r + 5) * b2 * b2 + s(r + 6) * b0 * b3 + s(r + 7) * b1 * b3 +
                                   s(r + 8) * b2 * b3 + s(r + 9) * b3 * b3);
    }
    if (!lsq6(s, 4)) return;
    for (int k = 0; k < 4; ++k) s(kBeta + k) += s(kX + k);
  }
}

// camera control points from the betas, camera points, sign, rotation and translation into s(kRt); mean reprojection error
D3R_HD_NOINLINE double compute_r_and_t(Scratch s, double fu, double fv, double uc, double vc) {
  for (int c = 0; c < 12; ++c) {
    double v = 0.0;
    for (int k = 0; k < 4; ++k) v += s(kBeta + k) * s(kNull + 12 * k + c);
    s(kCc + c) = v;
  }
  for (int i = 0; i < kSample; ++i)
    for (int d = 0; d < 3; ++d) {
      double v = 0.0;
      for (int j = 0; j < 4; ++j) v += s(kAlpha + 4 * i + j) * s(kCc + 3 * j + d);
      s(kPc + 3 * i + d) = v;
    }
  if (s(kPc + 2) < 0.0) {   // solve_for_sign
    for (int c = 0; c < 12; ++c) s(kCc + c) = -s(kCc + c);
    for (int c = 0; c < 15; ++c) s(kPc + c) = -s(kPc + c);
  }
  double pc0[3] = {0, 0, 0}, pw0[3] = {0, 0, 0};
  for (int i = 0; i < kSample; ++i)
D3R_UNROLL
    for (int d = 0; d < 3; ++d) {
      pc0[d] += s(kPc + 3 * i + d) / kSample;
      pw0[d] += s(kPw + 3 * i + d) / kSample;
    }
  // S[a][b] = sum (pw - pw0)_a (pc - pc0)_b; Horn's 4x4 N, its top eigenvector is the quaternion of the rotation pw -> pc
  double S[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (int i = 0; i < kSample; ++i)
D3R_UNROLL
    for (int a = 0; a < 3; ++a)
D3R_UNROLL
      for (int b = 0; b < 3; ++b) S[a][b] += (s(kPw + 3 * i + a) - pw0[a]) * (s(kPc + 3 * i + b) - pc0[b]);
  const double N[16] = {S[0][0] + S[1][1] + S[2][2], S[1][2] - S[2][1], S[2][0] - S[0][2], S[0][1] - S[1][0],
                        S[1][2] - S[2][1], S[0][0] - S[1][1] - S[2][2], S[0][1] + S[1][0], S[2][0] + S[0][2],
                        S[2][0] - S[0][2], S[0][1] + S[1][0], -S[0][0] + S[1][1] - S[2][2], S[1][2] + S[2][1],
                        S[0][1] - S[1][0], S[2][0] + S[0][2], S[1][2] + S[2][1], -S[0][0] - S[1][1] + S[2][2]};
D3R_UNROLL
  for (int k = 0; k < 16; ++k) s(kA + k) = N[k];
  jacobi(s, 4);
  int top = 0;
  for (int k = 1; k < 4; ++k)
    if (s(kA + 5 * k) > s(kA + 5 * top)) top = k;
  double w = s(kV + top), x = s(kV + 4 + top), y = s(kV + 8 + top), z = s(kV + 12 + top);
  const double qn = 1.0 / sqrt(w * w + x * x + y * y + z * z);
  w *= qn; x *= qn; y *= qn; z *= qn;
  const double R[9] = {w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y),
                       2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x),
                       2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z};
D3R_UNROLL
  for (int k = 0; k < 9; ++k) s(kRt + k) = R[k];
D3R_UNROLL
  for (int r = 0; r < 3; ++r) s(kRt + 9 + r) = pc0[r] - (R[3 * r] * pw0[0] + R[3 * r + 1] * pw0[1] + R[3 * r + 2] * pw0[2]);
  // epnp.cpp: reprojection_error
  double sum = 0.0;
  for (int i = 0; i < kSample; ++i) {
    const double X = s(kPw + 3 * i), Y = s(kPw + 3 * i + 1), Z = s(kPw + 3 * i + 2);
    const double Xc = R[0] * X + R[1] * Y + R[2] * Z + s(kRt + 9);
    const double Yc = R[3] * X + R[4] * Y + R[5] * Z + s(kRt + 10);
    const double iz = 1.0 / (R[6] * X + R[7] * Y + R[8] * Z + s(kRt + 11));
    const double du = s(kUv + 2 * i) - (uc + fu * Xc * iz), dv = s(kUv + 2 * i + 1) - (vc + fv * Yc * iz);
    sum += sqrt(du * du + dv * dv);
  }
  return sum / kSample;
}

// EPnP on the 5 points at s(kPw) / s(kUv); the pose of least reprojection error at s(kBest) = [R row-major | t].  False when
// the sample is degenerate (no finite pose).
D3R_HD_NOINLINE bool epnp(Scratch s, double fu, double fv, double uc, double vc) {
  // choose_control_points: centroid + PCA of the world points
  double c0[3] = {0, 0, 0};
  for (int i = 0; i < kSample; ++i)
D3R_UNROLL
    for (int d = 0; d < 3; ++d) c0[d] += s(kPw + 3 * i + d);
D3R_UNROLL
  for (int d = 0; d < 3; ++d) c0[d] /= kSample;
D3R_UNROLL
  for (int a = 0; a < 3; ++a)
D3R_UNROLL
    for (int b = 0; b < 3; ++b) {
      double v = 0.0;
      for (int i = 0; i < kSample; ++i) v += (s(kPw + 3 * i + a) - c0[a]) * (s(kPw + 3 * i + b) - c0[b]);
      s(kA + 3 * a + b) = v;
    }
  jacobi(s, 3);
  int ord[3] = {0, 1, 2};   // eigenvalues in decreasing order
D3R_UNROLL
  for (int i = 0; i < 3; ++i)
D3R_UNROLL
    for (int j = i + 1; j < 3; ++j)
      if (s(kA + 4 * ord[j]) > s(kA + 4 * ord[i])) {
        const int t = ord[i];
        ord[i] = ord[j];
        ord[j] = t;
      }
  const double lmax = s(kA + 4 * ord[0]);
  if (!(lmax > 0.0) || !isfinite(lmax)) return false;
  double e[3][3], sig[3];
D3R_UNROLL
  for (int k = 0; k < 3; ++k) {
    const double l = s(kA + 4 * ord[k]);
    sig[k] = l > kFlat * lmax ? sqrt(l / kSample) : 0.0;
D3R_UNROLL
    for (int d = 0; d < 3; ++d) e[k][d] = s(kV + 3 * d + ord[k]);
    // canonical sign: the component of largest magnitude (the first of equal ones) is positive
    int big = 0;
D3R_UNROLL
    for (int d = 1; d < 3; ++d)
      if (fabs(e[k][d]) > fabs(e[k][big])) big = d;
    const double sg = e[k][big] < 0.0 ? -1.0 : 1.0;
D3R_UNROLL
    for (int d = 0; d < 3; ++d) e[k][d] *= sg;
  }
D3R_UNROLL
  for (int d = 0; d < 3; ++d) s(kCw + d) = c0[d];
D3R_UNROLL
  for (int k = 0; k < 3; ++k)
D3R_UNROLL
    for (int d = 0; d < 3; ++d) s(kCw + 3 * (k + 1) + d) = c0[d] + sig[k] * e[k][d];
  // compute_barycentric_coordinates (CC is U diag(sig): its pseudo-inverse is diag(1/sig) U^T)
  for (int i = 0; i < kSample; ++i) {
    double a0 = 1.0;
D3R_UNROLL
    for (int k = 0; k < 3; ++k) {
      double p = 0.0;
D3R_UNROLL
      for (int d = 0; d < 3; ++d) p += e[k][d] * (s(kPw + 3 * i + d) - c0[d]);
      const double a = sig[k] > 0.0 ? p / sig[k] : 0.0;
      s(kAlpha + 4 * i + k + 1) = a;
      a0 -= a;
    }
    s(kAlpha + 4 * i) = a0;
  }
  // M^T M of the 10 x 12 M (fill_M): rows 2i: a_j fu, 0, a_j (uc - u_i); 2i + 1: 0, a_j fv, a_j (vc - v_i)
  for (int k = 0; k < 144; ++k) s(kA + k) = 0.0;
  for (int i = 0; i < kSample; ++i) {
    const double du = uc - s(kUv + 2 * i), dv = vc - s(kUv + 2 * i + 1);
    for (int r = 0; r < 2; ++r) {
      const int m = kL;   // one row of M, staged where L goes later
      for (int j = 0; j < 4; ++j) {
        const double a = s(kAlpha + 4 * i + j);
        s(m + 3 * j) = r == 0 ? a * fu : 0.0;
        s(m + 3 * j + 1) = r == 0 ? 0.0 : a * fv;
        s(m + 3 * j + 2) = a * (r == 0 ? du : dv);
      }
D3R_UNROLL_BY(1)
      for (int p = 0; p < 12; ++p) {
        const double mp = s(m + p);
D3R_UNROLL_BY(4)
        for (int q = 0; q < 12; ++q) s(kA + 12 * p + q) += mp * s(m + q);
      }
    }
  }
  jacobi(s, 12);
  // the four smallest eigenvalues' vectors, v[0] of the smallest (epnp.cpp: ut + 12 * 11, ut + 12 * 10, ...)
  int used = 0;
  for (int k = 0; k < 4; ++k) {
    int best = -1;
    for (int j = 0; j < 12; ++j)
      if (!((used >> j) & 1) && (best < 0 || s(kA + 13 * j) < s(kA + 13 * best))) best = j;
    if (best < 0) return false;
    used |= 1 << best;
    for (int c = 0; c < 12; ++c) s(kNull + 12 * k + c) = s(kV + 12 * c + best);
  }
  // canonical basis of span(v[0], v[1]): v[0] = P e / |P e| with e = kCanon (1, 2, ..., 12), v[1] = the unit vector orthogonal
  // to it in the plane (its sign does not change the pose)
  {
    double p0 = 0.0, p1 = 0.0;
    for (int c = 0; c < 12; ++c) {
      p0 += (c + 1) * s(kNull + c);
      p1 += (c + 1) * s(kNull + 12 + c);
    }
    const double r = sqrt(p0 * p0 + p1 * p1);
    if (!(r > 0.0)) return false;
    const double c0 = p0 / r, c1 = p1 / r;
    for (int c = 0; c < 12; ++c) {
      const double a = s(kNull + c), b = s(kNull + 12 + c);
      s(kNull + c) = c0 * a + c1 * b;
      s(kNull + 12 + c) = -c1 * a + c0 * b;
    }
  }
  // compute_L_6x10 and compute_rho
  for (int k = 0; k < 6; ++k) {
    int a, b;
    pair_of(k, a, b);
    double dv[4][3];
D3R_UNROLL
    for (int v = 0; v < 4; ++v)
D3R_UNROLL
      for (int d = 0; d < 3; ++d) dv[v][d] = s(kNull + 12 * v + 3 * a + d) - s(kNull + 12 * v + 3 * b + d);
    auto dot = [&](int p, int q) { return dv[p][0] * dv[q][0] + dv[p][1] * dv[q][1] + dv[p][2] * dv[q][2]; };
    const int r = kL + 10 * k;
    s(r + 0) = dot(0, 0);
    s(r + 1) = 2.0 * dot(0, 1);
    s(r + 2) = dot(1, 1);
    s(r + 3) = 2.0 * dot(0, 2);
    s(r + 4) = 2.0 * dot(1, 2);
    s(r + 5) = dot(2, 2);
    s(r + 6) = 2.0 * dot(0, 3);
    s(r + 7) = 2.0 * dot(1, 3);
    s(r + 8) = 2.0 * dot(2, 3);
    s(r + 9) = dot(3, 3);
    double rho = 0.0;
    for (int d = 0; d < 3; ++d) {
      const double t = s(kCw + 3 * a + d) - s(kCw + 3 * b + d);
      rho += t * t;
    }
    s(kRho + k) = rho;
  }
  // the three beta estimates (find_betas_approx_1/2/3), each refined by Gauss-Newton; least reprojection error wins
  double best_err = 0.0;
  bool have = false;
  for (int variant = 1; variant <= 3; ++variant) {
    const int ncol = variant == 1 ? 4 : (variant == 2 ? 3 : 5);
    for (int i = 0; i < 6; ++i) {
      for (int j = 0; j < ncol; ++j) {
        const int col = variant == 1 ? (j == 0 ? 0 : j == 1 ? 1 : j == 2 ? 3 : 6) : j;
        s(kQ + i * 5 + j) = s(kL + 10 * i + col);
      }
      s(kRhs + i) = s(kRho + i);
    }
    for (int k = 0; k < 4; ++k) s(kBeta + k) = 0.0;
    if (!lsq6(s, ncol)) continue;
    const double x0 = s(kX), x1 = s(kX + 1), x2 = s(kX + 2);
    if (variant == 1) {
      const double r = sqrt(fabs(x0));
      const double sg = x0 < 0.0 ? -1.0 : 1.0;
      s(kBeta) = r;
      for (int k = 1; k < 4; ++k) s(kBeta + k) = sg * s(kX + k) / r;
    } else {
      double b0 = sqrt(fabs(x0));
      const double b1 = x0 < 0.0 ? (x2 < 0.0 ? sqrt(-x2) : 0.0) : (x2 > 0.0 ? sqrt(x2) : 0.0);
      if (x1 < 0.0) b0 = -b0;
      s(kBeta) = b0;
      s(kBeta + 1) = b1;
      if (variant == 3) s(kBeta + 2) = s(kX + 3) / b0;
    }
    gauss_newton(s);
    const double err = compute_r_and_t(s, fu, fv, uc, vc);
    bool finite = isfinite(err);
    for (int k = 0; k < 12; ++k) finite &= isfinite(s(kRt + k));
    if (finite && (!have || err < best_err)) {
      have = true;
      best_err = err;
      for (int k = 0; k < 12; ++k) s(kBest + k) = s(kRt + k);
    }
  }
  return have;
}

// ---- scoring ----
struct Camera {
  double fx, fy, cx, cy;
};

// squared reprojection error of one correspondence in fp32, as OpenCV's PnP RANSAC callback computes it
D3R_HD float reproj_err2(const double Rt[12], const Camera& cam, float X, float Y, float Z, float u, float v) {
  const double x = dadd(dadd(dadd(dmul(Rt[0], X), dmul(Rt[1], Y)), dmul(Rt[2], Z)), Rt[9]);
  const double y = dadd(dadd(dadd(dmul(Rt[3], X), dmul(Rt[4], Y)), dmul(Rt[5], Z)), Rt[10]);
  double z = dadd(dadd(dadd(dmul(Rt[6], X), dmul(Rt[7], Y)), dmul(Rt[8], Z)), Rt[11]);
  z = z != 0.0 ? 1.0 / z : 1.0;
  const float pu = (float)dadd(dmul(dmul(x, z), cam.fx), cam.cx);
  const float pv = (float)dadd(dmul(dmul(y, z), cam.fy), cam.cy);
  const float du = fsub(u, pu), dv = fsub(v, pv);
  return fadd(fmul(du, du), fmul(dv, dv));
}

// ---- stopping rule ----
// calib3d/src/ptsetreg.cpp: RANSACUpdateNumIters
D3R_HD int update_num_iters(double p, double ep, int model_points, int max_iters) {
  p = p > 0.0 ? (p < 1.0 ? p : 1.0) : 0.0;
  ep = ep > 0.0 ? (ep < 1.0 ? ep : 1.0) : 0.0;
  double num = 1.0 - p;
  num = num > 2.2250738585072014e-308 ? num : 2.2250738585072014e-308;
  double denom = 1.0 - pow(1.0 - ep, (double)model_points);
  if (denom < 2.2250738585072014e-308) return 0;
  num = log(num);
  denom = log(denom);
  return denom >= 0.0 || -num >= max_iters * (-denom) ? max_iters : (int)rint(num / denom);
}

// The loop's state between rounds of hypotheses.
struct State {
  int32_t best;        // index of the best hypothesis, -1 while there is none
  int32_t best_count;  // its inlier count
  int32_t niters;      // current iteration bound
  int32_t evaluated;   // hypotheses the sequential loop has run
  int32_t done;        // 1 once the loop has ended
  int32_t pad;
  double pose[12];     // the best hypothesis' [R | t]
};

D3R_HD void state_init(State& st, int max_iters) {
  st.best = -1;
  st.best_count = 0;
  st.niters = max_iters > 1 ? max_iters : 1;
  st.evaluated = 0;
  st.done = 0;
  st.pad = 0;
  for (int k = 0; k < 12; ++k) st.pose[k] = 0.0;
}

// Runs the sequential loop over hypotheses h0 .. h0 + m - 1 with their counts (a count < 0 marks an invalid hypothesis) and
// poses.  With n == kSample there is one hypothesis and no scoring: valid means all 5 points are inliers.
D3R_HD void scan_round(State& st, int32_t h0, int32_t m, const int32_t* counts, const double* poses, int32_t n,
                           double confidence) {
  if (st.done) return;
  for (int32_t i = 0; i < m; ++i) {
    const int32_t h = h0 + i;
    int32_t c = counts[i];
    if (n == kSample) c = c >= 0 ? kSample : -1;
    if (c > (st.best_count > kSample - 1 ? st.best_count : kSample - 1)) {
      st.best = h;
      st.best_count = c;
      for (int k = 0; k < 12; ++k) st.pose[k] = poses[12 * i + k];
      st.niters = n == kSample ? 1 : update_num_iters(confidence, (double)(n - c) / n, kSample, st.niters);
    }
    if (n == kSample) st.niters = 1;
    if (h + 1 >= st.niters) {
      st.evaluated = h + 1;
      st.done = 1;
      return;
    }
  }
  st.evaluated = h0 + m;
}

}  // namespace pnp
}  // namespace d3r
