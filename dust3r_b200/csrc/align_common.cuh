// Shared code of the alignment kernels (csrc/align_step.cu: general CTA-per-chunk kernel; csrc/align_stream.cu:
// persistent warp-streaming kernel): workspace carving, fixed-point accumulation, quaternion / Adam math, the
// derived-transform refresh, the small-parameter step run by the last CTA of every iteration, and the iteration launch.
#pragma once
#include "d3r_common.cuh"
#include "pdl.cuh"
#include "prof.h"
#include "sm90_ptx.cuh"

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
  long long* ent_acc;    // [2E][13]  fixed-point (2^40) accumulators, zero between launches
  long long* img_acc;    // [n][12]
  long long* ovf;        // [1]       split iteration: partial-range overflow seen by the pixel pass (directly after img_acc, so
                         //           [ent_acc | img_acc | ovf] is one contiguous block that one all-reduce(SUM) carries)
  float* grad;           // [11n + 10E] multi-pass small-step scratch: raw gradients in the flat parameter layout
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
  w.ovf = reinterpret_cast<long long*>(ws + o); o += 4;
  w.grad = ws + o;     o += align4(int64_t(n) * 11 + int64_t(E) * 10);
  w.flags = reinterpret_cast<int*>(ws + o); o += 4;
  w.entT = ws + o;     o += align4(int64_t(2) * E * kEdgeT);
  w.geomE = ws + o;    o += align4(int64_t(E) * 24);
  w.geomI = ws + o;    o += align4(int64_t(n) * 20);
  return w;
}

// Where the block [ent_acc | img_acc | ovf] sits in the workspace (in floats) and how many int64 words it holds: what a
// multi-GPU caller all-reduces between the pixel pass and the small step of a split iteration.
inline void reduce_block(int n, int E, int64_t* offset_floats, int64_t* n_words) {
  *offset_floats = align4(int64_t(E) * kEdgeT) + align4(int64_t(n) * kImgT);
  *n_words = int64_t(2) * E * kEntVals + int64_t(n) * kImgVals + 1;
}

inline int64_t workspace_floats(int n, int E) {
  return align4(int64_t(E) * kEdgeT) + align4(int64_t(n) * kImgT) + align4(int64_t(2) * E * kEntVals * 2) +
         align4(int64_t(n) * kImgVals * 2) + 4 + align4(int64_t(n) * 11 + int64_t(E) * 10) + 4 +
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
// A launch whose sums left the range (or met a NaN / Inf) reports NaN instead of a finite loss and gradient: fix_add
// turns a NaN partial into an ordinary integer, so the sums themselves no longer show it.  The last CTA reads the flag
// with ld.global.cg after the grid ticket, like the accumulators, and ORs it with its own range checks.
__device__ __forceinline__ int overflow_seen(const Workspace& ws) { return __ldcg(ws.flags); }
__device__ __forceinline__ float nan_if(bool poison, float v) { return poison ? __int_as_float(0x7fffffff) : v; }

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

template <int N>
__device__ __forceinline__ void load_row(const float* __restrict__ src, float (&c)[N]) {
  const float4* c4 = reinterpret_cast<const float4*>(src);
#pragma unroll
  for (int k = 0; k < N / 4; ++k) { const float4 t = c4[k]; c[4 * k] = t.x; c[4 * k + 1] = t.y; c[4 * k + 2] = t.z; c[4 * k + 3] = t.w; }
}

// Derived transforms of edge e from its pairwise pose p8 and adaptors a0, a1: the edgeT row M = s*R*diag(adapt) (9),
// s*T (3); for the streaming kernel the same row negated once per entry in entT (both sides of the edge see the same
// transform, read without indirection); and the geometry cache the next small step reads instead of recomputing it.
__device__ __forceinline__ void edge_refresh(const d3r_align_desc& D, const Workspace& ws, int e, const float* p8, float a0, float a1,
                                             float mean_sigma, float log_base) {
  float c[kGeomE];   // R (9) ad (3) s T (3) qhat (4) |q| sg^2 exp|t| (3)
  float* R = c; float* ad = c + 9; float* T = c + 13;
  quat_to_R(p8, R, c + 16, c + 20);
  float s = expf(p8[7]);
  if (D.norm_pw_scale) s *= expf(log_base - mean_sigma);   // base_opt.py:178-184
  c[12] = s;
  // adaptors (base_opt.py:143-148): adapt3 = exp((cat(a0,a0,a1) - mean)/pw_break)
  ad[0] = a0; ad[1] = a0; ad[2] = a1;
  if (D.norm_pw_scale) {
    const float mu = (a0 + a0 + a1) / 3.f;
    ad[0] -= mu; ad[1] -= mu; ad[2] -= mu;
  }
#pragma unroll
  for (int b = 0; b < 3; ++b) ad[b] = expf(ad[b] / D.pw_break);
#pragma unroll
  for (int a = 0; a < 3; ++a) T[a] = signed_expm1f(p8[4 + a]);
  float o[kEdgeT];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) o[a * 3 + b] = s * R[a * 3 + b] * ad[b];
#pragma unroll
  for (int a = 0; a < 3; ++a) o[9 + a] = s * T[a];
#pragma unroll
  for (int k = 0; k < kEdgeT; ++k) ws.edgeT[e * kEdgeT + k] = o[k];
  if (D.stream_kernel) {
    const int ei = D.edge_ent[e * 2 + 0], ej = D.edge_ent[e * 2 + 1];
#pragma unroll
    for (int k = 0; k < kEdgeT; ++k) { ws.entT[int64_t(ei) * kEdgeT + k] = -o[k]; ws.entT[int64_t(ej) * kEdgeT + k] = -o[k]; }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float t = p8[4 + a];
    const float sg = (t > 0.f) - (t < 0.f);
    c[21 + a] = sg * sg * expf(fabsf(t));
  }
#pragma unroll
  for (int k = 0; k < kGeomE; ++k) ws.geomE[int64_t(e) * kGeomE + k] = c[k];
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

// Raw gradients of edge e -- pairwise pose (quaternion 4, translation 3, log-scale 1) and adaptors (2) -- from the sums
// of its two entries (si, sj: sum g (x) q (9), sum g (3)) and its cached geometry c (geomE row), written to `grad` in the
// flat parameter layout.  Returns dL/dlog-scale, whose mean over the edges (the coupling of the normalised scales) the
// Adam step subtracts.
__device__ __forceinline__ float edge_grad(const d3r_align_desc& D, const SmallLayout& L, int e, const float* si, const float* sj,
                                           const float* c, float* grad) {
  const float* R = c; const float* ad = c + 9; const float sc = c[12]; const float* T = c + 13; const float* qh = c + 16;
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
  ge[7] = dLds * sc;
  float gad[3];
#pragma unroll
  for (int b = 0; b < 3; ++b) gad[b] = dad[b] * ad[b] / D.pw_break;
  if (D.norm_pw_scale) { const float mu = (gad[0] + gad[1] + gad[2]) / 3.f; gad[0] -= mu; gad[1] -= mu; gad[2] -= mu; }
  ge[8] = gad[0] + gad[1];
  ge[9] = gad[2];
#pragma unroll
  for (int k = 0; k < 8; ++k) grad[L.pw + e * 8 + k] = ge[k];
  grad[L.adapt + e * 2 + 0] = ge[8];
  grad[L.adapt + e * 2 + 1] = ge[9];
  return dLds * sc;
}

// Raw gradients of image i -- pose (quaternion 4, translation 3), focals (2), principal point (2) -- from its sums
// S (sum G (x) c (9), sum G (3); overwritten) and its cached geometry c (geomI row), written to `grad` in the flat
// parameter layout.
__device__ __forceinline__ void image_grad(const d3r_align_desc& D, const SmallLayout& L, int i, float (&S)[kImgVals], const float* c,
                                           float* grad) {
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
  gi[7] = D.tied_focal ? gfx + gfy : gfx;     // one shared focal: both slots get the summed gradient and evolve identically
  gi[8] = D.tied_focal ? gfx + gfy : gfy;
  gi[9] = -10.f * gpx / c[17];
  gi[10] = -10.f * gpy / c[18];
#pragma unroll
  for (int k = 0; k < 7; ++k) grad[L.poses + i * 7 + k] = gi[k];
  grad[L.focals + i * 2 + 0] = gi[7]; grad[L.focals + i * 2 + 1] = gi[8];
  grad[L.pp + i * 2 + 0] = gi[9]; grad[L.pp + i * 2 + 1] = gi[10];
}

__device__ __forceinline__ bool is_log_scale(const SmallLayout& L, int idx) { return idx >= L.pw && idx < L.adapt && ((idx - L.pw) & 7) == 7; }

// Adam step of the trainable flat parameter idx with raw gradient g: returns the new value and updates the moments m, v.
// With norm_pw_scale the log-scales see the mean-coupling term of the normalisation.
__device__ __forceinline__ float adam_param(const d3r_align_desc& D, const SmallLayout& L, int idx, float p, float& m, float& v, float g,
                                            float coupling, float step_size, float bc2s) {
  if (is_log_scale(L, idx) && D.norm_pw_scale) g -= coupling;
  return adam_update(p, g, m, v, D.beta1, D.beta2, step_size, bc2s, D.adam_eps);
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
    edge_refresh(D, ws, e, p8, sm[L.adapt + e * 2 + 0], sm[L.adapt + e * 2 + 1], mean_sigma, log_base);
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

// Multi-pass small-parameter step: backward through the small parameters + Adam, run by the last CTA of the grid for any
// graph size and for eval_only.  Strided loops over edges / images / parameters, gradients through global scratch, the
// loss summed over the entries in order.  The geometry of every edge and image is read from the cache that
// prepare_kernel and every step's refresh keep current.
static __device__ __noinline__ void small_param_step(const d3r_align_desc& D, const Workspace& ws, int it, float* s_red) {
  const int n = D.n_imgs, E = D.n_edges;
  const SmallLayout L(n, E);
  float* __restrict__ sm = D.small;
  float* __restrict__ am = D.small_m;
  float* __restrict__ av = D.small_v;
  const uint8_t* __restrict__ tr = D.small_trainable;
  const float step_size = D.sched[it * 4 + 1], bc2s = D.sched[it * 4 + 2];

  // phase 0: loss (fixed order over entries), one barrier
  float lpart = 0.f;
  int bad = threadIdx.x == 0 ? overflow_seen(ws) : 0;
  for (int k = threadIdx.x; k < 2 * E; k += blockDim.x) lpart += fix_get(ws.ent_acc + k * kEntVals + 12, bad);
  const float loss = block_sum8(lpart, s_red);
  D3R_TSTAMP(0);

  // phase 1: gradients -> ws.grad.  edges on low thread ids, images on high thread ids (different warps).
  float coupl = 0.f;
  if (!D.eval_only) {
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
      const int ei = D.edge_ent[e * 2 + 0], ej = D.edge_ent[e * 2 + 1];
      float si[12], sj[12], c[kGeomE];
#pragma unroll
      for (int k = 0; k < 12; ++k) { si[k] = fix_get(ws.ent_acc + ei * kEntVals + k, bad); sj[k] = fix_get(ws.ent_acc + ej * kEntVals + k, bad); }
      load_row(ws.geomE + int64_t(e) * kGeomE, c);
      coupl += edge_grad(D, L, e, si, sj, c, ws.grad);
    }
    for (int r = 0, i = img_of_thread(0); i < n; i = img_of_thread(++r)) {
      float S[kImgVals], c[kGeomI];
#pragma unroll
      for (int k = 0; k < kImgVals; ++k) S[k] = fix_get(ws.img_acc + i * kImgVals + k, bad);
      load_row(ws.geomI + int64_t(i) * kGeomI, c);
      image_grad(D, L, i, S, c, ws.grad);
    }
  }
  fix_report(bad, ws.flags);
  const bool poison = __syncthreads_or(bad);
  if (threadIdx.x == 0) D.loss_out[it] = nan_if(poison, loss);
  D3R_TSTAMP(1);
  // zero the accumulators for the next launch (everything has been read above; barrier inside block_sum8)
  const float coupling = block_sum8(coupl, s_red + 16) / float(E);
  for (int k = threadIdx.x; k < 2 * E * kEntVals; k += blockDim.x) ws.ent_acc[k] = 0;
  for (int k = threadIdx.x; k < n * kImgVals; k += blockDim.x) ws.img_acc[k] = 0;
  if (D.eval_only) return;
  D3R_TSTAMP(2);

  // phase 2: Adam over the flat parameter vector
  for (int idx = threadIdx.x; idx < L.total; idx += blockDim.x) {
    if (!tr[idx]) continue;
    float m = am[idx], v = av[idx];
    sm[idx] = adam_param(D, L, idx, sm[idx], m, v, ws.grad[idx], coupling, step_size, bc2s);
    am[idx] = m;
    av[idx] = v;
  }
  D3R_TSTAMP(3);
  __syncthreads();
  compute_transforms(D, ws, s_red + 24);
  D3R_TSTAMP(4);
}


// Outputs of a gradient launch (d3r_align_loss_grad): the gradient-export instantiations of both pixel kernels write the
// per-pixel log-depth gradient to logd_grad in their depth stage, and their last CTA runs small_grad_step instead of the
// small-parameter step.
struct GradOut {
  float* logd_grad;     // [sum stride_i]
  float* small_grad;    // [11n + 10E] flat parameter layout
  float* entry_loss;    // [E][2] or nullptr
};

// Gradient export in place of the small-parameter step: the loss (same order as small_param_step, so bit-identical to
// eval_only), the raw gradients of every parameter written to go.small_grad with the log-scale coupling folded in -- the
// values adam_param would feed Adam -- and optionally the per-entry loss.  No Adam step, no refresh; the accumulators
// are cleared as after any launch.
static __device__ __noinline__ void small_grad_step(const d3r_align_desc& D, const Workspace& ws, GradOut go, float* s_red) {
  const int n = D.n_imgs, E = D.n_edges;
  const SmallLayout L(n, E);
  float lpart = 0.f;
  int bad = threadIdx.x == 0 ? overflow_seen(ws) : 0;
  for (int k = threadIdx.x; k < 2 * E; k += blockDim.x) lpart += fix_get(ws.ent_acc + k * kEntVals + 12, bad);
  const float loss = block_sum8(lpart, s_red);

  float coupl = 0.f;
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    const int ei = D.edge_ent[e * 2 + 0], ej = D.edge_ent[e * 2 + 1];
    float si[12], sj[12], c[kGeomE];
#pragma unroll
    for (int k = 0; k < 12; ++k) { si[k] = fix_get(ws.ent_acc + ei * kEntVals + k, bad); sj[k] = fix_get(ws.ent_acc + ej * kEntVals + k, bad); }
    if (go.entry_loss) {
      go.entry_loss[e * 2 + 0] = fix_get(ws.ent_acc + ei * kEntVals + 12, bad);
      go.entry_loss[e * 2 + 1] = fix_get(ws.ent_acc + ej * kEntVals + 12, bad);
    }
    load_row(ws.geomE + int64_t(e) * kGeomE, c);
    coupl += edge_grad(D, L, e, si, sj, c, go.small_grad);
  }
  for (int r = 0, i = img_of_thread(0); i < n; i = img_of_thread(++r)) {
    float S[kImgVals], c[kGeomI];
#pragma unroll
    for (int k = 0; k < kImgVals; ++k) S[k] = fix_get(ws.img_acc + i * kImgVals + k, bad);
    load_row(ws.geomI + int64_t(i) * kGeomI, c);
    image_grad(D, L, i, S, c, go.small_grad);
  }
  fix_report(bad, ws.flags);
  const bool poison = __syncthreads_or(bad);
  if (threadIdx.x == 0) D.loss_out[0] = nan_if(poison, loss);
  // every accumulator has been read (barrier inside block_sum8): fold in the coupling, clear for the next launch
  const float coupling = block_sum8(coupl, s_red + 16) / float(E);
  if (poison) {            // every gradient and entry loss of the launch is NaN (the barriers above ordered the writes)
    for (int k = threadIdx.x; k < L.total; k += blockDim.x) go.small_grad[k] = nan_if(true, 0.f);
    if (go.entry_loss)
      for (int k = threadIdx.x; k < 2 * E; k += blockDim.x) go.entry_loss[k] = nan_if(true, 0.f);
  } else if (D.norm_pw_scale) {
    for (int e = threadIdx.x; e < E; e += blockDim.x) go.small_grad[L.pw + e * 8 + 7] -= coupling;   // written by this thread above
  }
  for (int k = threadIdx.x; k < 2 * E * kEntVals; k += blockDim.x) ws.ent_acc[k] = 0;
  for (int k = threadIdx.x; k < n * kImgVals; k += blockDim.x) ws.img_acc[k] = 0;
}

// ---- latency-optimised small-parameter step for graphs with one thread per edge / per image (E, n <= blockDim) ----
// The tail of a 60-microsecond iteration is bound by the dependent instruction chain of whichever thread does the most,
// so the work is cut three ways:
//   A  one thread per edge / per image: accumulators + the cached geometry -> raw gradients, written to shared memory
//      in the flat parameter layout;
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
  int bad = tid == 0 ? overflow_seen(ws) : 0;
  if (has_e) {
    const int ei = D.edge_ent[e * 2 + 0], ej = D.edge_ent[e * 2 + 1];
    float c[kGeomE];
    load_row(ws.geomE + int64_t(e) * kGeomE, c);
    float si[13], sj[13];
#pragma unroll
    for (int k = 0; k < 13; ++k) { si[k] = fix_get(ws.ent_acc + ei * kEntVals + k, bad); sj[k] = fix_get(ws.ent_acc + ej * kEntVals + k, bad); }
#pragma unroll
    for (int k = 0; k < kEntVals; ++k) { ws.ent_acc[ei * kEntVals + k] = 0; ws.ent_acc[ej * kEntVals + k] = 0; }   // read: clear for the next launch
    lpart = si[12] + sj[12];
    coupl = edge_grad(D, L, e, si, sj, c, g_s);
  }
  if (has_i) {
    float c[kGeomI];
    load_row(ws.geomI + int64_t(i) * kGeomI, c);
    float S[kImgVals];
#pragma unroll
    for (int k = 0; k < kImgVals; ++k) S[k] = fix_get(ws.img_acc + i * kImgVals + k, bad);   // S[a*3+b] = sum G_a c_b ; S[9+a] = sum G_a
#pragma unroll
    for (int k = 0; k < kImgVals; ++k) ws.img_acc[i * kImgVals + k] = 0;
    image_grad(D, L, i, S, c, g_s);
  }
  fix_report(bad, ws.flags);
  lpart = warp_sum(lpart);
  coupl = warp_sum(coupl);
  if ((tid & 31) == 0) { s_red[tid >> 5] = lpart; s_red[8 + (tid >> 5)] = coupl; }
  D3R_TSTAMP(0);
  const bool poison = __syncthreads_or(bad);
  float loss = 0.f, coupling = 0.f;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) { loss += s_red[w]; coupling += s_red[8 + w]; }
  coupling /= float(E);
  if (tid == 0) D.loss_out[it] = nan_if(poison, loss);
  D3R_TSTAMP(1);

  // ---- stage B: Adam, one thread per parameter
  float snew = 0.f;
  for (int r = 0, idx = tid; idx < L.total; idx += nthr, ++r) {
    float p, m, v;
    uint8_t t;
    if (r < 2) { p = pp_[r & 1]; m = pm_[r & 1]; v = pv_[r & 1]; t = pt_[r & 1]; }
    else { p = sm[idx]; m = am[idx]; v = av[idx]; t = tr[idx]; }
    if (t) {
      p = adam_param(D, L, idx, p, m, v, g_s[idx], coupling, step_size, bc2s);
      sm[idx] = p; am[idx] = m; av[idx] = v;
    }
    p_s[idx] = p;
    if (is_log_scale(L, idx)) snew += p;
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
    edge_refresh(D, ws, e, p8, p_s[L.adapt + e * 2 + 0], p_s[L.adapt + e * 2 + 1], mean_sigma, log_base);
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

// Launches iterations [it_begin, it_end) of an iteration kernel, `grid` CTAs of `threads` each.  Every launch allows
// programmatic stream serialisation, so that its CTAs run their launch-independent prologue while the previous iteration's
// last CTA is still in its small-parameter step; the kernels call pdl::sync_with_predecessor() before they read what that
// step wrote.  The shared-memory opt-in is a per-device function attribute (a process may drive several GPUs), so it is
// set on every call; two CTAs per SM need the maximum carve-out.
template <typename Arg>
static int alignment_launch_config(void (*kernel)(d3r_align_desc, Arg), int grid, int threads, size_t smem, cudaStream_t st,
                                   cudaLaunchConfig_t& cfg, cudaLaunchAttribute& at) {
  D3R_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  D3R_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3((unsigned)threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &at;
  cfg.numAttrs = 1;
  return D3R_OK;
}

static int launch_iterations(void (*kernel)(d3r_align_desc, int), const d3r_align_desc* desc, int grid, int threads, size_t smem,
                             int it_begin, int it_end, cudaStream_t st) {
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute at;
  if (int rc = alignment_launch_config(kernel, grid, threads, smem, st, cfg, at)) return rc;
  for (int it = it_begin; it < it_end; ++it) D3R_CUDA(cudaLaunchKernelEx(&cfg, kernel, *desc, it));
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}

// One launch of a gradient-export kernel (same launch attributes as an iteration).
static int launch_gradient(void (*kernel)(d3r_align_desc, GradOut), const d3r_align_desc* desc, int grid, int threads, size_t smem,
                           const GradOut& go, cudaStream_t st) {
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute at;
  if (int rc = alignment_launch_config(kernel, grid, threads, smem, st, cfg, at)) return rc;
  D3R_CUDA(cudaLaunchKernelEx(&cfg, kernel, *desc, go));
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}

}  // namespace align
}  // namespace d3r
