// Shared device code of the alignment kernels (csrc/align_step.cu: general CTA-per-chunk kernel; csrc/align_stream.cu:
// persistent warp-streaming kernel): workspace carving, fixed-point accumulation, quaternion / Adam math, the
// derived-transform refresh and the small-parameter step run by the last CTA of every iteration.
#pragma once
#include "d3r_common.cuh"
#include "prof.h"

namespace d3r {
namespace align {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kPPT = 8;                    // pixels per thread
constexpr int kChunk = kThreads * kPPT;    // pixels per CTA
constexpr int kEntVals = 13;               // 9 (g (x) q) + 3 (g) + 1 (loss)
constexpr int kImgVals = 12;               // 9 (G (x) c) + 3 (G)
constexpr int kEdgeT = 12;                 // M = s*R*diag(adapt) (9) + s*T (3)
constexpr int kImgT = 16;                  // R (9) T (3) 1/fx 1/fy cx cy

struct Workspace {
  float* edgeT;          // [E][12]
  float* imgT;           // [n][16]
  long long* ent_acc;    // [2E][13]  fixed-point (2^44) accumulators, zero between launches
  long long* img_acc;    // [n][12]
  float* g_edge;         // [E][10]   small-step scratch: pairwise-pose / adaptor gradients
  float* g_img;          // [n][11]   pose (7) / focal (2) / pp (2) gradients
  int* flags;            // [4]       [0] = fixed-point overflow seen
  float* entT;           // [2E][12]  streaming kernel: -M (9), -t (3) of the entry's edge, indexed by entry (no indirection)
  float* geomE;          // [E][24]   cache for the next small step: R (9) ad (3) s T (3) qhat (4) |q| sg^2 exp|t| (3)
  float* geomI;          // [n][20]   R (9) qhat (4) |q| sg^2 exp|t| (3) exp(f/focal_break) (2) pad
};
constexpr int kGeomE = 24, kGeomI = 20;

__host__ __device__ inline int64_t align4(int64_t x) { return (x + 3) & ~int64_t(3); }

__host__ __device__ inline Workspace carve(float* ws, int n, int E) {
  Workspace w;
  int64_t o = 0;
  w.edgeT = ws + o;    o += align4(int64_t(E) * kEdgeT);
  w.imgT = ws + o;     o += align4(int64_t(n) * kImgT);
  w.ent_acc = reinterpret_cast<long long*>(ws + o); o += align4(int64_t(2) * E * kEntVals * 2);
  w.img_acc = reinterpret_cast<long long*>(ws + o); o += align4(int64_t(n) * kImgVals * 2);
  w.g_edge = ws + o;   o += align4(int64_t(E) * 10);
  w.g_img = ws + o;    o += align4(int64_t(n) * 11);
  w.flags = reinterpret_cast<int*>(ws + o); o += 4;
  w.entT = ws + o;     o += align4(int64_t(2) * E * kEdgeT);
  w.geomE = ws + o;    o += align4(int64_t(E) * 24);
  w.geomI = ws + o;    o += align4(int64_t(n) * 20);
  return w;
}

inline int64_t workspace_floats(int n, int E) {
  return align4(int64_t(E) * kEdgeT) + align4(int64_t(n) * kImgT) + align4(int64_t(2) * E * kEntVals * 2) +
         align4(int64_t(n) * kImgVals * 2) + align4(int64_t(E) * 10) + align4(int64_t(n) * 11) + 4 +
         align4(int64_t(2) * E * kEdgeT) + align4(int64_t(E) * 24) + align4(int64_t(n) * 20);
}

// Order-independent (hence deterministic) cross-CTA accumulation: every warp contributes its exactly-ordered fp32
// partial sum as a 2^40 fixed-point integer through a 64-bit integer atomic.  Resolution 9.1e-13 (the sums are O(1..100) and
// end up in fp32), range +-8.4e6.  Overflow is reported, not silently wrapped: a partial must stay below 2^18 (checked where it
// is added; also catches NaN / Inf) and a total below 2^22 (checked where it is read) -- 16 partials at the limit would be needed
// to wrap the accumulator unnoticed, versus 2 with the 2^44 scale of round 1.
constexpr double kFixScale = 1099511627776.0;        // 2^40
__device__ __forceinline__ void fix_add(long long* dst, float x, int* overflow_flag) {
  if (!(fabsf(x) < 262144.f)) *overflow_flag = 1;     // also catches NaN / Inf
  const long long q = __double2ll_rn(double(x) * kFixScale);
  atomicAdd(reinterpret_cast<unsigned long long*>(dst), static_cast<unsigned long long>(q));
}
// 2^-40 * q without FP64 (int64 -> double conversions are multi-pass on sm_90 and sit on the small step's critical path):
// q = hi * 2^32 + lo; hi * 2^-8 carries the value, lo * 2^-40 < 2^-8 the fraction below.
// `bad` collects the range check in a register: a conditional STORE per value would order the 26 accumulator loads of a thread
// behind one another (measured: +3.6 us on the small step); the caller reports once with fix_report.
__device__ __forceinline__ float fix_get(const long long* src, int& bad) {
  const long long q = __ldcg(src);
  const int hi = int(q >> 32);
  const unsigned lo = unsigned(q);
  const float v = fmaf(__uint2float_rn(lo), 9.094947017729282e-13f /* 2^-40 */, __int2float_rn(hi) * 3.90625e-3f /* 2^-8 */);
  bad |= !(fabsf(v) < 4194304.f);                     // |total| >= 2^22: out of the supported range
  return v;
}
__device__ __forceinline__ void fix_report(int bad, int* overflow_flag) {
  if (bad) *overflow_flag = 1;
}

// Grid ticket: release this CTA's accumulations / log-depth updates and acquire everybody else's in ONE operation by one
// thread (the CTA barrier before / after it extends both to the other threads by cumulativity).  What the last CTA then reads
// of other CTAs' work are the fixed-point accumulators, fetched with ld.global.cg (L2, where the atomics were performed), so no
// CTA-wide fence (1 us for 256 threads) is needed after the ticket.
__device__ __forceinline__ int grid_ticket(int* counter) {
  int old;
  asm volatile("atom.add.acq_rel.gpu.global.s32 %0, [%1], 1;" : "=r"(old) : "l"(counter) : "memory");
  return old;
}

// offsets inside the `small` parameter buffer
struct SmallLayout {
  int poses, focals, pp, pw, adapt, total;
  __host__ __device__ SmallLayout(int n, int E) {
    poses = 0; focals = n * 7; pp = focals + n * 2; pw = pp + n * 2; adapt = pw + E * 8; total = adapt + E * 2;
  }
};

__device__ __forceinline__ float signed_expm1f(float x) {
  float s = (x > 0.f) - (x < 0.f);
  return s * expm1f(fabsf(x));
}

// unit quaternion (x,y,z,w) -> rotation, row-major R[a*3+b]
__device__ __forceinline__ void quat_to_R(const float* q, float* R, float* qhat, float* nrm) {
  float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  float x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
  R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - w * z);       R[2] = 2.f * (x * z + w * y);
  R[3] = 2.f * (x * y + w * z);       R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - w * x);
  R[6] = 2.f * (x * z - w * y);       R[7] = 2.f * (y * z + w * x);       R[8] = 1.f - 2.f * (x * x + y * y);
  if (qhat) { qhat[0] = x; qhat[1] = y; qhat[2] = z; qhat[3] = w; }
  if (nrm) *nrm = n;
}

// dL/dq (raw, un-normalised) from D = dL/dR
__device__ __forceinline__ void quat_backward(const float* D, const float* qh, float n, float* gq) {
  float x = qh[0], y = qh[1], z = qh[2], w = qh[3];
  float gx = 2.f * (y * (D[1] + D[3]) + z * (D[2] + D[6]) - 2.f * x * (D[4] + D[8]) + w * (D[7] - D[5]));
  float gy = 2.f * (x * (D[1] + D[3]) + z * (D[5] + D[7]) - 2.f * y * (D[0] + D[8]) + w * (D[2] - D[6]));
  float gz = 2.f * (x * (D[2] + D[6]) + y * (D[5] + D[7]) - 2.f * z * (D[0] + D[4]) + w * (D[3] - D[1]));
  float gw = 2.f * (x * (D[7] - D[5]) + y * (D[2] - D[6]) + z * (D[3] - D[1]));
  float dot = gx * x + gy * y + gz * z + gw * w;
  gq[0] = (gx - x * dot) / n; gq[1] = (gy - y * dot) / n; gq[2] = (gz - z * dot) / n; gq[3] = (gw - w * dot) / n;
}

// torch.optim.Adam single-tensor math (lerp for exp_avg; mul+addcmul for exp_avg_sq; addcdiv)
__device__ __forceinline__ float adam_update(float p, float g, float& m, float& v, float beta1, float beta2,
                                             float step_size, float bc2_sqrt, float eps) {
  m = m + (1.f - beta1) * (g - m);
  v = v * beta2 + (1.f - beta2) * g * g;
  float denom = sqrtf(v) / bc2_sqrt + eps;
  return p - step_size * (m / denom);
}

// optional timeline instrumentation (debug aid): 4 x uint64 globaltimer stamps per CTA
static __device__ unsigned long long* g_align_dbg = nullptr;
__device__ __forceinline__ unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// small-step stamps follow the per-CTA (general kernel) / per-warp (streaming kernel) rows
#define D3R_TSTAMP(i) do { if (g_align_dbg && threadIdx.x == 0) g_align_dbg[4 * size_t(D.stream_kernel ? D.stream_grid * 8 : D.n_chunks) + (i)] = gtime(); } while (0)

// ---- derived transforms / small-parameter step (run by ONE CTA while the rest of the chip idles) ----------
// Written for latency: independent global loads are issued together, block reductions cost one barrier (every
// thread re-adds the 8 warp partials itself), pointers are __restrict__, and the edge work (low thread ids)
// and image work (high thread ids) run concurrently on different warps.
__device__ __forceinline__ float block_sum8(float v, float* slot /* 8 floats */) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) slot[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) t += slot[w];
  return t;
}

struct EdgeGeom {
  float R[9], T[3], ad[3], s, qh[4], qn;
};
__device__ __forceinline__ void edge_geom(const float* p8, float a0, float a1, const d3r_align_desc& D, float mean_sigma,
                                          float log_base, EdgeGeom& g) {
  quat_to_R(p8, g.R, g.qh, &g.qn);
  g.s = expf(p8[7]);
  if (D.norm_pw_scale) g.s *= expf(log_base - mean_sigma);
  g.ad[0] = a0; g.ad[1] = a0; g.ad[2] = a1;
  if (D.norm_pw_scale) {
    const float mu = (a0 + a0 + a1) / 3.f;
    g.ad[0] -= mu; g.ad[1] -= mu; g.ad[2] -= mu;
  }
#pragma unroll
  for (int b = 0; b < 3; ++b) g.ad[b] = expf(g.ad[b] / D.pw_break);
#pragma unroll
  for (int a = 0; a < 3; ++a) g.T[a] = signed_expm1f(p8[4 + a]);
}

// what the next small step needs of an edge's / image's geometry (recomputing it there sits on the critical path)
__device__ __forceinline__ void store_geom_edge(float* __restrict__ c, const EdgeGeom& g, const float* p8) {
#pragma unroll
  for (int k = 0; k < 9; ++k) c[k] = g.R[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) { c[9 + k] = g.ad[k]; c[13 + k] = g.T[k]; }
  c[12] = g.s;
#pragma unroll
  for (int k = 0; k < 4; ++k) c[16 + k] = g.qh[k];
  c[20] = g.qn;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float t = p8[4 + a];
    const float sg = (t > 0.f) - (t < 0.f);
    c[21 + a] = sg * sg * expf(fabsf(t));
  }
}
__device__ __forceinline__ void image_transform_row(const d3r_align_desc& D, const float* q7, float f0, float f1, float pp0, float pp1,
                                                    int Hh, int Ww, float* __restrict__ o, float* __restrict__ c) {
  float R[9], qh[4], qn;
  quat_to_R(q7, R, qh, &qn);
#pragma unroll
  for (int k = 0; k < 9; ++k) { o[k] = R[k]; c[k] = R[k]; }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float t = q7[4 + a];
    const float sg = (t > 0.f) - (t < 0.f);
    o[9 + a] = signed_expm1f(t);
    c[14 + a] = sg * sg * expf(fabsf(t));
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) c[9 + k] = qh[k];
  c[13] = qn;
  const float ef0 = expf(f0 / D.focal_break), ef1 = expf(f1 / D.focal_break);
  c[17] = ef0; c[18] = ef1; c[19] = 0.f;
  o[12] = 1.f / ef0;
  o[13] = 1.f / ef1;
  o[14] = 0.5f * float(Ww) + 10.f * pp0;
  o[15] = 0.5f * float(Hh) + 10.f * pp1;
}

// image i is handled by thread (blockDim-1-i) so that images and edges land on different warps
__device__ __forceinline__ int img_of_thread(int it) { return int(blockDim.x) - 1 - int(threadIdx.x) + it * int(blockDim.x); }

static __device__ void compute_transforms(const d3r_align_desc& D, const Workspace& ws, float* s_red) {
  const int n = D.n_imgs, E = D.n_edges;
  const SmallLayout L(n, E);
  const float* __restrict__ sm = D.small;
  float part = 0.f;
  for (int e = threadIdx.x; e < E; e += blockDim.x) part += sm[L.pw + e * 8 + 7];
  const float mean_sigma = block_sum8(part, s_red) / float(E);   // base_opt.py:178-184
  const float log_base = logf(D.base_scale);
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    float p8[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) p8[k] = sm[L.pw + e * 8 + k];
    const float a0 = sm[L.adapt + e * 2 + 0], a1 = sm[L.adapt + e * 2 + 1];
    EdgeGeom g;
    edge_geom(p8, a0, a1, D, mean_sigma, log_base, g);
    float* o = ws.edgeT + e * kEdgeT;
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) o[a * 3 + b] = g.s * g.R[a * 3 + b] * g.ad[b];
#pragma unroll
    for (int a = 0; a < 3; ++a) o[9 + a] = g.s * g.T[a];
    if (D.stream_kernel) {   // the streaming kernel reads -M, -t per ENTRY (both sides of the edge see the same transform)
#pragma unroll
      for (int side = 0; side < 2; ++side) {
        float* oe = ws.entT + int64_t(D.edge_ent[e * 2 + side]) * kEdgeT;
#pragma unroll
        for (int k = 0; k < kEdgeT; ++k) oe[k] = -o[k];
      }
    }
    store_geom_edge(ws.geomE + int64_t(e) * kGeomE, g, p8);
  }
  for (int r = 0, i = img_of_thread(0); i < n; i = img_of_thread(++r)) {
    float p7[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) p7[k] = sm[L.poses + i * 7 + k];
    const float f0 = sm[L.focals + i * 2 + 0], f1 = sm[L.focals + i * 2 + 1];
    const float pp0 = sm[L.pp + i * 2 + 0], pp1 = sm[L.pp + i * 2 + 1];
    const int Hh = D.img_hw[i * 2 + 0], Ww = D.img_hw[i * 2 + 1];
    image_transform_row(D, p7, f0, f1, pp0, pp1, Hh, Ww, ws.imgT + i * kImgT, ws.geomI + int64_t(i) * kGeomI);
  }
}

// backward through the small parameters + Adam; run by the last CTA of the grid
static __device__ __noinline__ void small_param_step(const d3r_align_desc& D, const Workspace& ws, int it, float* s_red) {
  const int n = D.n_imgs, E = D.n_edges;
  const SmallLayout L(n, E);
  float* __restrict__ sm = D.small;
  float* __restrict__ am = D.small_m;
  float* __restrict__ av = D.small_v;
  const uint8_t* __restrict__ tr = D.small_trainable;
  const float step_size = D.sched[it * 4 + 1], bc2s = D.sched[it * 4 + 2];
  const float b1 = D.beta1, b2 = D.beta2, eps = D.adam_eps;

  // phase 0: loss (fixed order over entries) and mean log-scale, one barrier
  float lpart = 0.f, spart = 0.f;
  int bad = 0;
  for (int k = threadIdx.x; k < 2 * E; k += blockDim.x) lpart += fix_get(ws.ent_acc + k * kEntVals + 12, bad);
  for (int e = threadIdx.x; e < E; e += blockDim.x) spart += sm[L.pw + e * 8 + 7];
  lpart = warp_sum(lpart);
  spart = warp_sum(spart);
  if ((threadIdx.x & 31) == 0) { s_red[threadIdx.x >> 5] = lpart; s_red[8 + (threadIdx.x >> 5)] = spart; }
  __syncthreads();
  float loss = 0.f, mean_sigma = 0.f;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) { loss += s_red[w]; mean_sigma += s_red[8 + w]; }
  mean_sigma /= float(E);
  if (threadIdx.x == 0) D.loss_out[it] = loss;
  const float log_base = logf(D.base_scale);
  D3R_TSTAMP(0);

  // phase 1: gradients -> scratch.  edges on low thread ids, images on high thread ids (different warps).
  float coupl = 0.f;
  if (!D.eval_only) {
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
      float p8[8], si[12], sj[12];
      const int ei = D.edge_ent[e * 2 + 0], ej = D.edge_ent[e * 2 + 1];
#pragma unroll
      for (int k = 0; k < 8; ++k) p8[k] = sm[L.pw + e * 8 + k];
      const float a0 = sm[L.adapt + e * 2 + 0], a1 = sm[L.adapt + e * 2 + 1];
#pragma unroll
      for (int k = 0; k < 12; ++k) { si[k] = fix_get(ws.ent_acc + ei * kEntVals + k, bad); sj[k] = fix_get(ws.ent_acc + ej * kEntVals + k, bad); }
      EdgeGeom g;
      edge_geom(p8, a0, a1, D, mean_sigma, log_base, g);
      float dM[9], dt[3];
#pragma unroll
      for (int k = 0; k < 9; ++k) dM[k] = -(si[k] + sj[k]);   // dL/dM_ab = -sum g_a q_b
#pragma unroll
      for (int a = 0; a < 3; ++a) dt[a] = -(si[9 + a] + sj[9 + a]);
      float dLds = 0.f, dR[9], dad[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int b = 0; b < 3; ++b) {
          dLds += dM[a * 3 + b] * g.R[a * 3 + b] * g.ad[b];
          dR[a * 3 + b] = dM[a * 3 + b] * g.s * g.ad[b];
          dad[b] += dM[a * 3 + b] * g.s * g.R[a * 3 + b];
        }
        dLds += dt[a] * g.T[a];
      }
      float gr[10];
      quat_backward(dR, g.qh, g.qn, gr);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const float t = p8[4 + a];
        const float sg = (t > 0.f) - (t < 0.f);
        gr[4 + a] = dt[a] * g.s * sg * sg * expf(fabsf(t));
      }
      gr[7] = dLds * g.s;             // the mean-coupling term is subtracted in phase 2
      coupl += dLds * g.s;
      // adaptors (base_opt.py:143-148): adapt3 = exp((cat(a0,a0,a1) - mean)/pw_break)
      float gad[3];
#pragma unroll
      for (int b = 0; b < 3; ++b) gad[b] = dad[b] * g.ad[b] / D.pw_break;
      if (D.norm_pw_scale) { const float mu = (gad[0] + gad[1] + gad[2]) / 3.f; gad[0] -= mu; gad[1] -= mu; gad[2] -= mu; }
      gr[8] = gad[0] + gad[1];
      gr[9] = gad[2];
#pragma unroll
      for (int k = 0; k < 10; ++k) ws.g_edge[e * 10 + k] = gr[k];
    }
    for (int r = 0, i = img_of_thread(0); i < n; i = img_of_thread(++r)) {
      float q7[7], S[12];
#pragma unroll
      for (int k = 0; k < 7; ++k) q7[k] = sm[L.poses + i * 7 + k];
      const float f0 = sm[L.focals + i * 2 + 0], f1 = sm[L.focals + i * 2 + 1];
#pragma unroll
      for (int k = 0; k < 12; ++k) S[k] = fix_get(ws.img_acc + i * kImgVals + k, bad);   // S[a*3+b] = sum G_a c_b ; S[9+a] = sum G_a
      float R[9], qh[4], qn;
      quat_to_R(q7, R, qh, &qn);
      if (D.stream_kernel) {
        // the streaming kernel accumulates sum G (x) Y with Y = X - T = R c (world frame): sum G (x) c = (sum G (x) Y) R
        float Sc[9];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int b = 0; b < 3; ++b) Sc[a * 3 + b] = S[a * 3 + 0] * R[0 * 3 + b] + S[a * 3 + 1] * R[1 * 3 + b] + S[a * 3 + 2] * R[2 * 3 + b];
#pragma unroll
        for (int k = 0; k < 9; ++k) S[k] = Sc[k];
      }
      float gr[11];
      quat_backward(S, qh, qn, gr);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const float t = q7[4 + a];
        const float sg = (t > 0.f) - (t < 0.f);
        gr[4 + a] = S[9 + a] * sg * sg * expf(fabsf(t));
      }
      // focals: c_x = d (u-cx)/fx, fx = exp(phi/focal_break);  pp: cx = W/2 + 10 pp_x
      float gfx = 0.f, gfy = 0.f, gpx = 0.f, gpy = 0.f;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        gfx += R[a * 3 + 0] * S[a * 3 + 0];
        gfy += R[a * 3 + 1] * S[a * 3 + 1];
        gpx += R[a * 3 + 0] * S[a * 3 + 2];
        gpy += R[a * 3 + 1] * S[a * 3 + 2];
      }
      gfx = -gfx / D.focal_break;
      gfy = -gfy / D.focal_break;
      // one shared focal: both slots get the summed gradient and evolve identically
      gr[7] = D.tied_focal ? gfx + gfy : gfx;
      gr[8] = D.tied_focal ? gfx + gfy : gfy;
      gr[9] = -10.f * gpx / expf(f0 / D.focal_break);
      gr[10] = -10.f * gpy / expf(f1 / D.focal_break);
#pragma unroll
      for (int k = 0; k < 11; ++k) ws.g_img[i * 11 + k] = gr[k];
    }
  }
  fix_report(bad, ws.flags);
  D3R_TSTAMP(1);
  // zero the accumulators for the next launch (everything has been read above; barrier inside block_sum8)
  const float coupling = block_sum8(coupl, s_red + 16) / float(E);
  for (int k = threadIdx.x; k < 2 * E * kEntVals; k += blockDim.x) ws.ent_acc[k] = 0;
  for (int k = threadIdx.x; k < n * kImgVals; k += blockDim.x) ws.img_acc[k] = 0;
  if (D.eval_only) return;
  D3R_TSTAMP(2);

  // phase 2: Adam over the flat parameter vector  [poses 7n | focals 2n | pp 2n | pw 8E | adapt 2E]
  for (int idx = threadIdx.x; idx < L.total; idx += blockDim.x) {
    if (!tr[idx]) continue;
    float g;
    if (idx < L.focals) {
      const int i = idx / 7;
      g = ws.g_img[i * 11 + (idx - i * 7)];
    } else if (idx < L.pp) {
      const int r = idx - L.focals;
      g = ws.g_img[(r >> 1) * 11 + 7 + (r & 1)];
    } else if (idx < L.pw) {
      const int r = idx - L.pp;
      g = ws.g_img[(r >> 1) * 11 + 9 + (r & 1)];
    } else if (idx < L.adapt) {
      const int r = idx - L.pw;
      g = ws.g_edge[(r >> 3) * 10 + (r & 7)];
      if ((r & 7) == 7 && D.norm_pw_scale) g -= coupling;
    } else {
      const int r = idx - L.adapt;
      g = ws.g_edge[(r >> 1) * 10 + 8 + (r & 1)];
    }
    float m = am[idx], v = av[idx];
    sm[idx] = adam_update(sm[idx], g, m, v, b1, b2, step_size, bc2s, eps);
    am[idx] = m;
    av[idx] = v;
  }
  D3R_TSTAMP(3);
  __syncthreads();
  compute_transforms(D, ws, s_red + 24);
  D3R_TSTAMP(4);
}


// ---- latency-optimised small-parameter step for graphs with one thread per edge / per image (E, n <= blockDim) ----
// Same mathematics as small_param_step.  The tail of a 60-microsecond iteration is bound by the dependent instruction
// chain of whichever thread does the most, so the work is cut three ways:
//   A  one thread per edge / per image: accumulators + the geometry CACHED by the previous refresh (ws.geomE / geomI:
//      rotation, normalised quaternion, scale, adaptors ... -- nothing is recomputed) -> raw gradients, written to
//      shared memory in the flat parameter layout;
//   B  one thread per PARAMETER: Adam (parameter, moments and flag were requested before stage A, so their latency is
//      hidden behind it), refreshed value to global and shared memory;
//   C  one thread per edge / per image again: derived transforms + geometry cache of the refreshed parameters.
// Two block barriers; loss, mean-coupling and the refreshed mean log-scale ride on them.  `scr` is the CTA's dynamic
// shared memory (idle by now), >= 2 * (11 n + 10 E) floats.
static __device__ __forceinline__ void small_param_step_fast(const d3r_align_desc& D, int it, float* s_red, float* scr) {
  const int n = D.n_imgs, E = D.n_edges;
  const Workspace ws = carve(D.workspace, n, E);   // recomputed here: a reference would be read back from the caller's stack (DRAM by now)
  const SmallLayout L(n, E);
  float* __restrict__ sm = D.small;
  float* __restrict__ am = D.small_m;
  float* __restrict__ av = D.small_v;
  const uint8_t* __restrict__ tr = D.small_trainable;
  const float step_size = D.sched[it * 4 + 1], bc2s = D.sched[it * 4 + 2];
  const float b1 = D.beta1, b2 = D.beta2, eps = D.adam_eps;
  float* g_s = scr;               // [L.total] raw gradients
  float* p_s = scr + L.total;     // [L.total] refreshed parameters
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int e = tid, i = nthr - 1 - tid;
  const bool has_e = e < E, has_i = i < n;

  // stage-B operands of this thread's first two parameters: requested now, consumed after stage A
  float pp_[2], pm_[2], pv_[2];
  uint8_t pt_[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int idx = tid + r * nthr;
    pt_[r] = 0;
    if (idx < L.total) { pp_[r] = sm[idx]; pm_[r] = am[idx]; pv_[r] = av[idx]; pt_[r] = tr[idx]; }
  }

  // ---- stage A
  float lpart = 0.f, coupl = 0.f;
  int bad = 0;
  if (has_e) {
    const int ei = D.edge_ent[e * 2 + 0], ej = D.edge_ent[e * 2 + 1];
    float c[kGeomE];
    const float4* c4 = reinterpret_cast<const float4*>(ws.geomE + int64_t(e) * kGeomE);
#pragma unroll
    for (int k = 0; k < kGeomE / 4; ++k) { const float4 t = c4[k]; c[4 * k] = t.x; c[4 * k + 1] = t.y; c[4 * k + 2] = t.z; c[4 * k + 3] = t.w; }
    float si[13], sj[13];
#pragma unroll
    for (int k = 0; k < 13; ++k) { si[k] = fix_get(ws.ent_acc + ei * kEntVals + k, bad); sj[k] = fix_get(ws.ent_acc + ej * kEntVals + k, bad); }
#pragma unroll
    for (int k = 0; k < kEntVals; ++k) { ws.ent_acc[ei * kEntVals + k] = 0; ws.ent_acc[ej * kEntVals + k] = 0; }   // read: clear for the next launch
    lpart = si[12] + sj[12];
    const float* R = c; const float* ad = c + 9; const float sc = c[12]; const float* T = c + 13; const float* qh = c + 16;
    float dM[9], dt[3];
#pragma unroll
    for (int k = 0; k < 9; ++k) dM[k] = -(si[k] + sj[k]);
#pragma unroll
    for (int a = 0; a < 3; ++a) dt[a] = -(si[9 + a] + sj[9 + a]);
    float dLds = 0.f, dR[9], dad[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        dLds += dM[a * 3 + b] * R[a * 3 + b] * ad[b];
        dR[a * 3 + b] = dM[a * 3 + b] * sc * ad[b];
        dad[b] += dM[a * 3 + b] * sc * R[a * 3 + b];
      }
      dLds += dt[a] * T[a];
    }
    float ge[10];
    quat_backward(dR, qh, c[20], ge);
#pragma unroll
    for (int a = 0; a < 3; ++a) ge[4 + a] = dt[a] * sc * c[21 + a];
    ge[7] = dLds * sc;             // the mean-coupling term is subtracted in stage B
    coupl = dLds * sc;
    float gad[3];
#pragma unroll
    for (int b = 0; b < 3; ++b) gad[b] = dad[b] * ad[b] / D.pw_break;
    if (D.norm_pw_scale) { const float mu = (gad[0] + gad[1] + gad[2]) / 3.f; gad[0] -= mu; gad[1] -= mu; gad[2] -= mu; }
    ge[8] = gad[0] + gad[1];
    ge[9] = gad[2];
#pragma unroll
    for (int k = 0; k < 8; ++k) g_s[L.pw + e * 8 + k] = ge[k];
    g_s[L.adapt + e * 2 + 0] = ge[8];
    g_s[L.adapt + e * 2 + 1] = ge[9];
  }
  if (has_i) {
    float c[kGeomI];
    const float4* c4 = reinterpret_cast<const float4*>(ws.geomI + int64_t(i) * kGeomI);
#pragma unroll
    for (int k = 0; k < kGeomI / 4; ++k) { const float4 t = c4[k]; c[4 * k] = t.x; c[4 * k + 1] = t.y; c[4 * k + 2] = t.z; c[4 * k + 3] = t.w; }
    float S[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) S[k] = fix_get(ws.img_acc + i * kImgVals + k, bad);   // S[a*3+b] = sum G_a c_b ; S[9+a] = sum G_a
#pragma unroll
    for (int k = 0; k < kImgVals; ++k) ws.img_acc[i * kImgVals + k] = 0;
    const float* R = c;
    if (D.stream_kernel) {   // the streaming kernel accumulates sum G (x) Y, Y = R c: sum G (x) c = (sum G (x) Y) R
      float Sc[9];
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) Sc[a * 3 + b] = S[a * 3 + 0] * R[0 * 3 + b] + S[a * 3 + 1] * R[1 * 3 + b] + S[a * 3 + 2] * R[2 * 3 + b];
#pragma unroll
      for (int k = 0; k < 9; ++k) S[k] = Sc[k];
    }
    float gi[11];
    quat_backward(S, c + 9, c[13], gi);
#pragma unroll
    for (int a = 0; a < 3; ++a) gi[4 + a] = S[9 + a] * c[14 + a];
    float gfx = 0.f, gfy = 0.f, gpx = 0.f, gpy = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      gfx += R[a * 3 + 0] * S[a * 3 + 0];
      gfy += R[a * 3 + 1] * S[a * 3 + 1];
      gpx += R[a * 3 + 0] * S[a * 3 + 2];
      gpy += R[a * 3 + 1] * S[a * 3 + 2];
    }
    gfx = -gfx / D.focal_break;
    gfy = -gfy / D.focal_break;
    gi[7] = D.tied_focal ? gfx + gfy : gfx;     // one shared focal: both slots get the summed gradient
    gi[8] = D.tied_focal ? gfx + gfy : gfy;
    gi[9] = -10.f * gpx / c[17];
    gi[10] = -10.f * gpy / c[18];
#pragma unroll
    for (int k = 0; k < 7; ++k) g_s[L.poses + i * 7 + k] = gi[k];
    g_s[L.focals + i * 2 + 0] = gi[7]; g_s[L.focals + i * 2 + 1] = gi[8];
    g_s[L.pp + i * 2 + 0] = gi[9]; g_s[L.pp + i * 2 + 1] = gi[10];
  }
  fix_report(bad, ws.flags);
  lpart = warp_sum(lpart);
  coupl = warp_sum(coupl);
  if ((tid & 31) == 0) { s_red[tid >> 5] = lpart; s_red[8 + (tid >> 5)] = coupl; }
  D3R_TSTAMP(0);
  __syncthreads();
  float loss = 0.f, coupling = 0.f;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) { loss += s_red[w]; coupling += s_red[8 + w]; }
  coupling /= float(E);
  if (tid == 0) D.loss_out[it] = loss;
  D3R_TSTAMP(1);

  // ---- stage B: Adam, one thread per parameter
  float snew = 0.f;
  for (int r = 0, idx = tid; idx < L.total; idx += nthr, ++r) {
    float p, m, v;
    uint8_t t;
    if (r < 2) { p = pp_[r & 1]; m = pm_[r & 1]; v = pv_[r & 1]; t = pt_[r & 1]; }
    else { p = sm[idx]; m = am[idx]; v = av[idx]; t = tr[idx]; }
    const bool is_sigma = idx >= L.pw && idx < L.adapt && ((idx - L.pw) & 7) == 7;
    if (t) {
      float g = g_s[idx];
      if (is_sigma && D.norm_pw_scale) g -= coupling;
      p = adam_update(p, g, m, v, b1, b2, step_size, bc2s, eps);
      sm[idx] = p; am[idx] = m; av[idx] = v;
    }
    p_s[idx] = p;
    if (is_sigma) snew += p;
  }
  snew = warp_sum(snew);
  if ((tid & 31) == 0) s_red[16 + (tid >> 5)] = snew;
  D3R_TSTAMP(2);
  __syncthreads();
  float mean_sigma = 0.f;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) mean_sigma += s_red[16 + w];
  mean_sigma /= float(E);                                   // base_opt.py:178-184
  const float log_base = logf(D.base_scale);
  D3R_TSTAMP(3);

  // ---- stage C: derived transforms + geometry cache of the refreshed parameters
  if (has_e) {
    float p8[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) p8[k] = p_s[L.pw + e * 8 + k];
    EdgeGeom g;
    edge_geom(p8, p_s[L.adapt + e * 2 + 0], p_s[L.adapt + e * 2 + 1], D, mean_sigma, log_base, g);
    float o[kEdgeT];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) o[a * 3 + b] = g.s * g.R[a * 3 + b] * g.ad[b];
#pragma unroll
    for (int a = 0; a < 3; ++a) o[9 + a] = g.s * g.T[a];
#pragma unroll
    for (int k = 0; k < kEdgeT; ++k) ws.edgeT[e * kEdgeT + k] = o[k];
    if (D.stream_kernel) {
      const int ei = D.edge_ent[e * 2 + 0], ej = D.edge_ent[e * 2 + 1];
#pragma unroll
      for (int k = 0; k < kEdgeT; ++k) { ws.entT[int64_t(ei) * kEdgeT + k] = -o[k]; ws.entT[int64_t(ej) * kEdgeT + k] = -o[k]; }
    }
    store_geom_edge(ws.geomE + int64_t(e) * kGeomE, g, p8);
  }
  if (has_i) {
    float q7[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) q7[k] = p_s[L.poses + i * 7 + k];
    image_transform_row(D, q7, p_s[L.focals + i * 2 + 0], p_s[L.focals + i * 2 + 1], p_s[L.pp + i * 2 + 0], p_s[L.pp + i * 2 + 1],
                        D.img_hw[i * 2 + 0], D.img_hw[i * 2 + 1], ws.imgT + i * kImgT, ws.geomI + int64_t(i) * kGeomI);
  }
  D3R_TSTAMP(4);
}

// The small step's inputs were last touched one iteration (>= 200 MB of streaming) ago: by the time the last CTA wants them
// they are in DRAM and every dependent load costs a microsecond (measured: 4.9 us for the first round trip, 2.8 us for the
// second).  Every CTA therefore asks the L2 for them when it runs out of pixels -- a few dozen lines, L2 hits for all but
// the first CTA -- so that the last CTA finds them next to the accumulators.
__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2::evict_last [%0];" ::"l"(p));
}
__device__ __forceinline__ void prefetch_range(const void* base, int64_t bytes, int tid, int nthr) {
  const char* p = reinterpret_cast<const char*>(base);
  for (int64_t o = int64_t(tid) * 128; o < bytes; o += int64_t(nthr) * 128) prefetch_l2(p + o);
}
__device__ __forceinline__ bool fast_small_step_applies(const d3r_align_desc& D, int scr_floats) {
  return !D.eval_only && D.n_edges <= int(blockDim.x) && D.n_imgs <= int(blockDim.x) && 2 * (11 * D.n_imgs + 10 * D.n_edges) <= scr_floats;
}
static __device__ __forceinline__ void prefetch_small_step_inputs(const d3r_align_desc& D, const Workspace& ws, int it, int scr_floats,
                                                                  int tid, int nthr) {
  if (!fast_small_step_applies(D, scr_floats)) return;
  const int n = D.n_imgs, E = D.n_edges, total = 11 * n + 10 * E;
  prefetch_range(D.small, int64_t(total) * 4, tid, nthr);
  prefetch_range(D.small_m, int64_t(total) * 4, tid, nthr);
  prefetch_range(D.small_v, int64_t(total) * 4, tid, nthr);
  prefetch_range(D.small_trainable, total, tid, nthr);
  prefetch_range(ws.geomE, int64_t(E) * kGeomE * 4, tid, nthr);
  prefetch_range(ws.geomI, int64_t(n) * kGeomI * 4, tid, nthr);
  prefetch_range(D.edge_ent, int64_t(E) * 8, tid, nthr);
  prefetch_range(D.img_hw, int64_t(n) * 8, tid, nthr);
  if (tid == 0) prefetch_l2(D.sched + it * 4);
}

// dispatcher used by both iteration kernels
// `scr` / `scr_floats`: the CTA's dynamic shared memory, free once its pixels are done
static __device__ __forceinline__ void small_step(const d3r_align_desc& D, const Workspace& ws, int it, float* s_red, float* scr,
                                                  int scr_floats) {
  if (fast_small_step_applies(D, scr_floats))
    small_param_step_fast(D, it, s_red, scr);
  else
    small_param_step(D, ws, it, s_red);
}

}  // namespace align
}  // namespace d3r
