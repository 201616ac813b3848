// Evaluation criteria of the reference's training code (dust3r/losses.py: Regr3D and its shift / scale-invariant variants, L21,
// ConfLoss) on the GPU, without a host round trip between stages, and the segmented masked median they are built on.
//
// A batch is B pairs x two views.  Pair b is one segment: its n1 view-1 pixels followed by its n2 view-2 pixels, the order of
// the reference's torch.cat((view1, view2), dim=1).  The per-pixel passes tile each view of each segment into slots of kChunk
// pixels (one CTA each, grid = (slots of view 1 + slots of view 2, B)), so that no CTA straddles a view or a segment:
//   1. prepare   gt <- inv(camera_pose of view 1) * gt, the valid mask (& |gt| <= dist_clip), and per slot the fp64 sums of
//                |gt| and |pred| over the valid pixels and their count (the 'avg_dis' normalisation);
//   2. norm      per segment, the fixed-order sum of its slots -> the two normalisation factors;
//   3. medians   (shift-invariant) z of gt and pred; (scale-invariant) x, y, z of gt and pred, then |p - centre| of each: every
//                stage writes its columns, invalid pixels as NaN, and runs the segmented median below on all of them at once;
//   4. loss      normalisation, shift and scale applied in registers, the L2 distance, conf * l - alpha * log(conf), per slot
//                fp64 sums; with reduction 'none' the distances of the valid pixels are written compacted in the order of
//                tensor[mask] (row-major over B, H, W of each view) from an exclusive prefix of the per-slot counts;
//   5. final     per view, the fixed-order sum of its slots -> the fp32 results the Python side returns.
// All sums are per-CTA partials reduced in a fixed order, so two calls on the same inputs give the same bits.
//
// Segmented median: torch.nanmedian semantics (element (n - 1) / 2 of the sorted non-NaN values, NaN for a row without one) by a
// radix select on order-preserving uint32 keys, most significant 8-bit digit first: per digit, one histogram launch over all
// rows (shared-memory bins, warp-aggregated, then integer atomics into the row's global bins) and one select launch (a CTA per
// row walks the 256 bins to the digit that holds the wanted rank).  Integer counts make the result independent of the order
// the atomics land in.  The key order puts -0 below +0; torch compares them equal, so either may be returned where they tie.
#include "d3r_common.cuh"
#include "prof.h"

#include <cmath>

namespace d3r {
namespace crit {

constexpr int kThreads = 256;
constexpr int kPerThread = 16;
constexpr int kChunk = kThreads * kPerThread;   // pixels of one slot / elements of one histogram CTA
constexpr int kBins = 256;
constexpr int kPasses = 4;

// d3r_criterion flags
constexpr int kNorm = 1, kGtScale = 2, kShift = 4, kScale = 8, kConf = 16, kClip = 32;

// per-segment parameters: P[field * B + b]
enum Field { kNfGt = 0, kNfPr, kShiftGt, kShiftPr, kCentreGt, kCentrePr = kCentreGt + 3, kScaleGt = kCentrePr + 3, kScalePr, kFields };

__device__ __forceinline__ uint32_t float_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct MedianState {
  uint32_t prefix;   // digits fixed so far
  uint32_t rank;     // rank of the wanted element among the keys that share the prefix
  int32_t empty;     // no non-NaN value in the row
  int32_t pad;
};

__global__ void __launch_bounds__(kThreads) median_hist_kernel(const float* __restrict__ vals, long long len, int pass,
                                                               const MedianState* __restrict__ state, uint32_t* __restrict__ hist) {
  const int s = blockIdx.y;
  const int shift = 24 - 8 * pass;
  uint32_t prefix = 0;
  if (pass > 0) {
    const MedianState st = state[s];
    if (st.empty) return;
    prefix = st.prefix >> (shift + 8);
  }
  __shared__ uint32_t bins[kBins];
  for (int i = threadIdx.x; i < kBins; i += kThreads) bins[i] = 0;
  __syncthreads();
  const float* row = vals + (long long)s * len;
  const long long base = (long long)blockIdx.x * kChunk;
  const unsigned lane = threadIdx.x & 31;
#pragma unroll 4
  for (int j = 0; j < kPerThread; ++j) {
    const long long i = base + j * kThreads + threadIdx.x;
    int bin = -1;
    if (i < len) {
      const float v = row[i];
      if (!isnan(v)) {
        const uint32_t k = float_key(v);
        if (pass == 0 || (k >> (shift + 8)) == prefix) bin = (k >> shift) & 0xff;
      }
    }
    // lanes with the same bin add once: the leading digits of nearby values mostly agree
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    if (bin >= 0 && lane == (unsigned)(__ffs(peers) - 1)) atomicAdd(&bins[bin], (uint32_t)__popc(peers));
  }
  __syncthreads();
  uint32_t* out = hist + ((long long)pass * gridDim.y + s) * kBins;
  for (int i = threadIdx.x; i < kBins; i += kThreads)
    if (bins[i]) atomicAdd(&out[i], bins[i]);
}

// one CTA per row: inclusive scan of the 256 bins, the digit whose range holds the rank
__global__ void __launch_bounds__(kBins) median_select_kernel(int pass, int n_seg, MedianState* __restrict__ state,
                                                              const uint32_t* __restrict__ hist, float* __restrict__ out) {
  const int s = blockIdx.x;
  MedianState st = pass == 0 ? MedianState{0u, 0u, 0, 0} : state[s];
  if (st.empty) return;
  __shared__ uint32_t scan[kBins];
  __shared__ uint32_t total;
  const uint32_t h = hist[((long long)pass * n_seg + s) * kBins + threadIdx.x];
  scan[threadIdx.x] = h;
  __syncthreads();
  for (int o = 1; o < kBins; o <<= 1) {   // Hillis-Steele
    const uint32_t v = threadIdx.x >= o ? scan[threadIdx.x - o] : 0u;
    __syncthreads();
    scan[threadIdx.x] += v;
    __syncthreads();
  }
  if (threadIdx.x == kBins - 1) total = scan[kBins - 1];
  __syncthreads();
  if (pass == 0) {
    if (total == 0) {
      if (threadIdx.x == 0) {
        state[s] = MedianState{0u, 0u, 1, 0};
        out[s] = __int_as_float(0x7fc00000);
      }
      return;
    }
    st.rank = (total - 1) / 2;
  }
  const uint32_t before = scan[threadIdx.x] - h;
  if (h > 0 && st.rank >= before && st.rank < before + h) {   // exactly one thread
    st.prefix |= (uint32_t)threadIdx.x << (24 - 8 * pass);
    st.rank -= before;
    state[s] = st;
    if (pass == kPasses - 1) out[s] = key_float(st.prefix);
  }
}

struct MedianLayout {
  long long hist, state, bytes;
  explicit MedianLayout(long long n_seg) {
    hist = 0;
    state = hist + ((long long)kPasses * n_seg * kBins * 4 + 255) / 256 * 256;
    bytes = state + (n_seg * (long long)sizeof(MedianState) + 255) / 256 * 256;
  }
};

static void median_launch(int n_seg, long long len, const float* vals, float* out, char* ws, cudaStream_t st) {
  const MedianLayout lay(n_seg);
  uint32_t* hist = reinterpret_cast<uint32_t*>(ws + lay.hist);
  MedianState* state = reinterpret_cast<MedianState*>(ws + lay.state);
  cudaMemsetAsync(hist, 0, (size_t)kPasses * n_seg * kBins * 4, st);
  const dim3 grid((unsigned)((len + kChunk - 1) / kChunk), (unsigned)n_seg);
  for (int p = 0; p < kPasses; ++p) {
    median_hist_kernel<<<grid, kThreads, 0, st>>>(vals, len, p, state, hist);
    median_select_kernel<<<n_seg, kBins, 0, st>>>(p, n_seg, state, hist, out);
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// criteria

struct Args {
  int B, c1, c2, flags;
  long long n1, n2;
  const float* T;                 // [B][16] inv(camera_pose of view 1), row-major
  const float* gt[2];             // [B][n][3]
  const uint8_t* valid[2];        // [B][n]
  const float* pr[2];             // [B][n][3]
  const float* conf[2];           // [B][n] (kConf)
  float clip, alpha;
  const float* P;                 // [kFields][B]
};

struct Pix {
  float g[3], p[3];
  bool valid;
};

enum Stage { kRaw = 0, kNormed, kShifted, kScaled };

// pixel i of view v of segment b with the transforms up to `stage` applied, in the reference's order of operations
template <int kStage>
__device__ __forceinline__ Pix load_pixel(const Args& a, int b, int v, long long i) {
  const long long n = v ? a.n2 : a.n1;
  const long long q = (long long)b * n + i;
  const float* T = a.T + b * 16;
  const float* gs = (v ? a.gt[1] : a.gt[0]) + 3 * q;   // a ternary keeps the parameter arrays out of local memory
  const float x = gs[0], y = gs[1], z = gs[2];
  Pix r;
#pragma unroll
  for (int k = 0; k < 3; ++k) r.g[k] = T[4 * k] * x + T[4 * k + 1] * y + T[4 * k + 2] * z + T[4 * k + 3];
  r.valid = (v ? a.valid[1] : a.valid[0])[q] != 0;
  if (a.flags & kClip) r.valid = r.valid && sqrtf(r.g[0] * r.g[0] + r.g[1] * r.g[1] + r.g[2] * r.g[2]) <= a.clip;
  const float* ps = (v ? a.pr[1] : a.pr[0]) + 3 * q;
  r.p[0] = ps[0]; r.p[1] = ps[1]; r.p[2] = ps[2];
  const int B = a.B;
  if (kStage >= kNormed && (a.flags & kNorm)) {
    const float fp = a.P[kNfPr * B + b];
#pragma unroll
    for (int k = 0; k < 3; ++k) r.p[k] = r.p[k] / fp;
    if (!(a.flags & kGtScale)) {
      const float fg = a.P[kNfGt * B + b];
#pragma unroll
      for (int k = 0; k < 3; ++k) r.g[k] = r.g[k] / fg;
    }
  }
  if (kStage >= kShifted && (a.flags & kShift)) {
    r.g[2] -= a.P[kShiftGt * B + b];
    r.p[2] -= a.P[kShiftPr * B + b];
  }
  if (kStage >= kScaled && (a.flags & kScale)) {
    const float sg = a.P[kScaleGt * B + b];
    float sp = a.P[kScalePr * B + b];
    if (!isnan(sp)) sp = fminf(fmaxf(sp, 1e-3f), 1e3f);   // torch.clip keeps NaN
    if (a.flags & kGtScale) {
      const float f = sg / sp;
#pragma unroll
      for (int k = 0; k < 3; ++k) r.p[k] *= f;
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        r.g[k] = r.g[k] / sg;
        r.p[k] = r.p[k] / sp;
      }
    }
  }
  return r;
}

__device__ __forceinline__ float norm3(const float* v) { return sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

// fixed-order sum of N doubles over the CTA; the result is valid in thread 0
template <int N>
__device__ __forceinline__ void block_sum(double (&v)[N]) {
  __shared__ double s[N][kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    double x = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (lane == 0) s[k][warp] = x;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      double x = 0.0;
      for (int w = 0; w < kThreads / 32; ++w) x += s[k][w];
      v[k] = x;
    }
  }
}

// (slot of blockIdx) -> view, first pixel, pixel count of the view
__device__ __forceinline__ void slot_of_block(const Args& a, int& v, long long& base, long long& n) {
  v = (int)blockIdx.x >= a.c1;
  base = (long long)(v ? blockIdx.x - a.c1 : blockIdx.x) * kChunk;
  n = v ? a.n2 : a.n1;
}

// per slot {sum |gt|, sum |pred|, count} over its valid pixels
__global__ void __launch_bounds__(kThreads) prepare_kernel(Args a, double* __restrict__ part) {
  int v;
  long long base, n;
  slot_of_block(a, v, base, n);
  const int b = blockIdx.y;
  double acc[3] = {0.0, 0.0, 0.0};
  for (int j = 0; j < kPerThread; ++j) {
    const long long i = base + j * kThreads + threadIdx.x;
    if (i >= n) break;
    const Pix px = load_pixel<kRaw>(a, b, v, i);
    if (px.valid) {
      acc[0] += norm3(px.g);
      acc[1] += norm3(px.p);
      acc[2] += 1.0;
    }
  }
  block_sum<3>(acc);
  if (threadIdx.x == 0) {
    double* o = part + 3 * ((long long)b * (a.c1 + a.c2) + blockIdx.x);
    o[0] = acc[0]; o[1] = acc[1]; o[2] = acc[2];
  }
}

// normalize_pointcloud(..., 'avg_dis'): per segment sum |p| / (count + 1e-8), clipped below at 1e-8 (NaN kept)
__global__ void __launch_bounds__(kThreads) norm_kernel(Args a, const double* __restrict__ part, float* __restrict__ P) {
  const int b = blockIdx.x, ns = a.c1 + a.c2;
  double acc[3] = {0.0, 0.0, 0.0};
  for (int x = threadIdx.x; x < ns; x += kThreads) {
    const double* o = part + 3 * ((long long)b * ns + x);
    acc[0] += o[0]; acc[1] += o[1]; acc[2] += o[2];
  }
  block_sum<3>(acc);
  if (threadIdx.x == 0) {
    for (int k = 0; k < 2; ++k) {
      float f = acc[2] > 0.0 ? (float)(acc[k] / acc[2]) : 0.f;
      if (f < 1e-8f) f = 1e-8f;
      P[(k == 0 ? kNfGt : kNfPr) * a.B + b] = f;
    }
  }
}

// median columns of one stage, [col][B][n1 + n2], NaN at invalid pixels
enum Columns { kDepth = 0, kCentre, kRadius };

template <int kWhat>
__global__ void __launch_bounds__(kThreads) columns_kernel(Args a, float* __restrict__ cols) {
  const int b = blockIdx.y;
  const long long L = a.n1 + a.n2;
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= L) return;
  const int v = i >= a.n1;
  const Pix px = load_pixel<kWhat == kDepth ? kNormed : kShifted>(a, b, v, v ? i - a.n1 : i);
  const float nan = __int_as_float(0x7fc00000);
  const long long col = (long long)a.B * L;
  float* o = cols + (long long)b * L + i;
  if (kWhat == kDepth) {            // depth shift: z
    o[0] = px.valid ? px.g[2] : nan;
    o[col] = px.valid ? px.p[2] : nan;
  } else if (kWhat == kCentre) {    // centre: x, y, z
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      o[k * col] = px.valid ? px.g[k] : nan;
      o[(3 + k) * col] = px.valid ? px.p[k] : nan;
    }
  } else {                          // scale: |p - centre| (the centre medians are in P)
    float dg[3], dp[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      dg[k] = px.g[k] - a.P[(kCentreGt + k) * a.B + b];
      dp[k] = px.p[k] - a.P[(kCentrePr + k) * a.B + b];
    }
    o[0] = px.valid ? norm3(dg) : nan;
    o[col] = px.valid ? norm3(dp) : nan;
  }
}

// exclusive prefix of the per-slot valid counts, view by view in tensor[mask] order (b-major, then slot)
__global__ void offsets_kernel(Args a, const double* __restrict__ part, long long* __restrict__ off) {
  const int v = threadIdx.x;
  if (v > 1) return;
  const int ns = a.c1 + a.c2, c = v ? a.c2 : a.c1, x0 = v ? a.c1 : 0;
  long long run = 0;
  for (int b = 0; b < a.B; ++b)
    for (int x = x0; x < x0 + c; ++x) {
      const long long s = (long long)b * ns + x;
      off[s] = run;
      run += (long long)part[3 * s + 2];
    }
}

// per slot {sum l, sum conf * l - alpha * log(conf), count}; with pix: compacted distances, with mask_out: the valid mask
__global__ void __launch_bounds__(kThreads) loss_kernel(Args a, double* __restrict__ part, const long long* __restrict__ off,
                                                        float* pix0, float* pix1, uint8_t* mask0, uint8_t* mask1) {
  int v;
  long long base, n;
  slot_of_block(a, v, base, n);
  const int b = blockIdx.y;
  const long long slot = (long long)b * (a.c1 + a.c2) + blockIdx.x;
  float* pix = v ? pix1 : pix0;
  uint8_t* mask = v ? mask1 : mask0;
  __shared__ int wcount[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long run = pix ? off[slot] : 0;
  double acc[3] = {0.0, 0.0, 0.0};
  for (int j = 0; j < kPerThread; ++j) {
    const long long i = base + j * kThreads + threadIdx.x;
    if (base + j * kThreads >= n) break;   // uniform over the CTA
    bool valid = false;
    float l = 0.f;
    if (i < n) {
      const Pix px = load_pixel<kScaled>(a, b, v, i);
      valid = px.valid;
      if (mask) mask[(long long)b * n + i] = valid ? 1 : 0;
      if (valid) {
        const float d[3] = {px.p[0] - px.g[0], px.p[1] - px.g[1], px.p[2] - px.g[2]};
        l = norm3(d);
        acc[0] += l;
        acc[2] += 1.0;
        if (a.flags & kConf) {
          const float c = (v ? a.conf[1] : a.conf[0])[(long long)b * n + i];
          acc[1] += c * l - a.alpha * logf(c);
        }
      }
    }
    if (pix) {   // block-wide exclusive scan of the valid flags, in pixel order
      const unsigned bal = __ballot_sync(0xffffffffu, valid);
      if (lane == 0) wcount[warp] = __popc(bal);
      __syncthreads();
      int before = 0, total = 0;
      for (int w = 0; w < kThreads / 32; ++w) {
        before += w < warp ? wcount[w] : 0;
        total += wcount[w];
      }
      if (valid) pix[run + before + __popc(bal & ((1u << lane) - 1u))] = l;
      run += total;
      __syncthreads();
    }
  }
  block_sum<3>(acc);
  if (threadIdx.x == 0) {
    double* o = part + 3 * slot;
    o[0] = acc[0]; o[1] = acc[1]; o[2] = acc[2];
  }
}

// out[0..1] per-view distance (mean, sum, or with reduction 'none' the mean / NaN the details report), out[2..3] per-view
// confidence loss (mean, 0 for an empty view), out[4] the criterion's value, out[5..6] the valid counts (int32 bits)
__global__ void __launch_bounds__(kThreads) final_kernel(Args a, const double* __restrict__ part, int reduction, float* __restrict__ out) {
  const int ns = a.c1 + a.c2;
  float r[4];
  int cnt[2];
  for (int v = 0; v < 2; ++v) {
    const int c = v ? a.c2 : a.c1, x0 = v ? a.c1 : 0;
    double acc[3] = {0.0, 0.0, 0.0};
    for (long long q = threadIdx.x; q < (long long)a.B * c; q += kThreads) {
      const double* o = part + 3 * ((q / c) * ns + x0 + q % c);
      acc[0] += o[0]; acc[1] += o[1]; acc[2] += o[2];
    }
    block_sum<3>(acc);
    __syncthreads();
    if (threadIdx.x == 0) {
      const bool any = acc[2] > 0.0;
      if (reduction == 1) r[v] = (float)acc[0];
      else r[v] = any ? (float)(acc[0] / acc[2]) : (reduction == 2 ? __int_as_float(0x7fc00000) : 0.f);
      r[2 + v] = any ? (float)(acc[1] / acc[2]) : 0.f;
      cnt[v] = (int)acc[2];
    }
  }
  if (threadIdx.x == 0) {
    out[0] = r[0]; out[1] = r[1]; out[2] = r[2]; out[3] = r[3];
    out[4] = (a.flags & kConf) ? r[2] + r[3] : (reduction == 2 ? __int_as_float(0x7fc00000) : r[0] + r[1]);
    out[5] = __int_as_float(cnt[0]);
    out[6] = __int_as_float(cnt[1]);
  }
}

// tests/test_criterion_float64_gpu.py reads P back: the first kFields * B floats of the workspace, in enum Field order
struct Layout {
  long long P, part_prep, part_loss, off, cols, med, bytes;
  int ncols;
  Layout(int B, long long n1, long long n2, int flags) {
    const long long ns = (long long)B * ((n1 + kChunk - 1) / kChunk + (n2 + kChunk - 1) / kChunk);
    ncols = (flags & kScale) ? 6 : (flags & kShift) ? 2 : 0;
    auto up = [](long long x) { return (x + 255) / 256 * 256; };
    P = 0;
    part_prep = P + up(4ll * kFields * B);
    part_loss = part_prep + up(24 * ns);
    off = part_loss + up(24 * ns);
    cols = off + up(8 * ns);
    med = cols + up(4ll * ncols * B * (n1 + n2));
    bytes = med + (ncols ? MedianLayout((long long)ncols * B).bytes : 0);
  }
};

}  // namespace crit
}  // namespace d3r

using namespace d3r::crit;

extern "C" int64_t d3r_nanmedian_workspace_bytes(int32_t n_seg) { return n_seg > 0 ? MedianLayout(n_seg).bytes : 0; }

extern "C" int d3r_segmented_nanmedian(int32_t n_seg, int64_t seg_len, const float* vals_dev, float* out_dev, void* workspace_dev,
                                       int64_t workspace_bytes, void* stream) {
  D3R_CHECK_ARG(vals_dev && out_dev && workspace_dev, "d3r_segmented_nanmedian: null pointer");
  D3R_CHECK_ARG(n_seg > 0 && n_seg <= 65535, "d3r_segmented_nanmedian: n_seg = %d outside [1, 65535]", n_seg);
  D3R_CHECK_ARG(seg_len > 0 && seg_len < (1ll << 32), "d3r_segmented_nanmedian: seg_len = %lld outside [1, 2^32)", (long long)seg_len);
  D3R_CHECK_ARG(workspace_bytes >= MedianLayout(n_seg).bytes, "d3r_segmented_nanmedian: workspace of %lld bytes, need %lld",
                (long long)workspace_bytes, MedianLayout(n_seg).bytes);
  cudaStream_t st = (cudaStream_t)stream;
  d3r::prof::Scope scope("segmented_nanmedian", st, 0.0, 4.0 * kPasses * double(n_seg) * seg_len, 2 * kPasses);
  median_launch(n_seg, seg_len, vals_dev, out_dev, static_cast<char*>(workspace_dev), st);
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}

extern "C" int64_t d3r_criterion_workspace_bytes(int32_t B, int64_t n1, int64_t n2, int32_t flags) {
  return B > 0 && n1 > 0 && n2 > 0 ? Layout(B, n1, n2, flags).bytes : 0;
}

extern "C" int d3r_criterion(int32_t B, int64_t n1, int64_t n2, int32_t flags, int32_t reduction, float dist_clip, float alpha,
                             const float* T_dev, const float* gt1_dev, const float* gt2_dev, const uint8_t* valid1_dev,
                             const uint8_t* valid2_dev, const float* pr1_dev, const float* pr2_dev, const float* conf1_dev,
                             const float* conf2_dev, float* out_dev, float* pix1_dev, float* pix2_dev, uint8_t* mask1_dev,
                             uint8_t* mask2_dev, void* workspace_dev, int64_t workspace_bytes, void* stream) {
  D3R_CHECK_ARG(T_dev && gt1_dev && gt2_dev && valid1_dev && valid2_dev && pr1_dev && pr2_dev && out_dev && workspace_dev,
                "d3r_criterion: null pointer");
  D3R_CHECK_ARG(!(flags & kConf) || (conf1_dev && conf2_dev), "d3r_criterion: confidence weighting needs conf1 and conf2");
  D3R_CHECK_ARG(!(flags & ~63), "d3r_criterion: unknown flags %#x", flags);
  D3R_CHECK_ARG(reduction >= 0 && reduction <= 2, "d3r_criterion: reduction %d not in {0 mean, 1 sum, 2 none}", reduction);
  D3R_CHECK_ARG(!pix1_dev == !pix2_dev && !mask1_dev == !mask2_dev && (!pix1_dev || reduction == 2),
                "d3r_criterion: per-pixel outputs come in pairs, and only with reduction 'none'");
  D3R_CHECK_ARG(B > 0 && B <= 65535 && n1 > 0 && n2 > 0, "d3r_criterion: B = %d, n1 = %lld, n2 = %lld", B, (long long)n1, (long long)n2);
  const int c1 = (int)((n1 + kChunk - 1) / kChunk), c2 = (int)((n2 + kChunk - 1) / kChunk);
  D3R_CHECK_ARG((long long)B * (n1 + n2) < (1ll << 31) && 6ll * B <= 65535,
                "d3r_criterion: %d pairs of %lld + %lld pixels exceed the supported range", B, (long long)n1, (long long)n2);
  const Layout lay(B, n1, n2, flags);
  D3R_CHECK_ARG(workspace_bytes >= lay.bytes, "d3r_criterion: workspace of %lld bytes, need %lld (d3r_criterion_workspace_bytes)",
                (long long)workspace_bytes, lay.bytes);
  char* ws = static_cast<char*>(workspace_dev);
  float* P = reinterpret_cast<float*>(ws + lay.P);
  double* part_prep = reinterpret_cast<double*>(ws + lay.part_prep);
  double* part_loss = reinterpret_cast<double*>(ws + lay.part_loss);
  long long* off = reinterpret_cast<long long*>(ws + lay.off);
  float* cols = reinterpret_cast<float*>(ws + lay.cols);
  char* med = ws + lay.med;

  Args a;
  a.B = B; a.c1 = c1; a.c2 = c2; a.flags = flags; a.n1 = n1; a.n2 = n2;
  a.T = T_dev;
  a.gt[0] = gt1_dev; a.gt[1] = gt2_dev;
  a.valid[0] = valid1_dev; a.valid[1] = valid2_dev;
  a.pr[0] = pr1_dev; a.pr[1] = pr2_dev;
  a.conf[0] = conf1_dev; a.conf[1] = conf2_dev;
  a.clip = dist_clip; a.alpha = alpha;
  a.P = P;

  cudaStream_t st = (cudaStream_t)stream;
  const long long L = n1 + n2;
  const double px = double(B) * L;
  const int launches = 4 + (pix1_dev ? 1 : 0) + ((flags & kShift) ? 1 + 2 * kPasses : 0) + ((flags & kScale) ? 2 * (1 + 2 * kPasses) : 0);
  d3r::prof::Scope scope("criterion", st, 0.0, px * (2 * 29.0 + (flags & kScale ? 5 * 4 * (kPasses + 2.0) : 0.0)), launches);
  const dim3 slots((unsigned)(c1 + c2), (unsigned)B), cgrid((unsigned)((L + kThreads - 1) / kThreads), (unsigned)B);
  prepare_kernel<<<slots, kThreads, 0, st>>>(a, part_prep);
  norm_kernel<<<B, kThreads, 0, st>>>(a, part_prep, P);
  if (flags & kShift) {
    columns_kernel<kDepth><<<cgrid, kThreads, 0, st>>>(a, cols);
    median_launch(2 * B, L, cols, P + kShiftGt * B, med, st);
  }
  if (flags & kScale) {
    columns_kernel<kCentre><<<cgrid, kThreads, 0, st>>>(a, cols);
    median_launch(6 * B, L, cols, P + kCentreGt * B, med, st);
    columns_kernel<kRadius><<<cgrid, kThreads, 0, st>>>(a, cols);
    median_launch(2 * B, L, cols, P + kScaleGt * B, med, st);
  }
  if (pix1_dev) offsets_kernel<<<1, 32, 0, st>>>(a, part_prep, off);
  loss_kernel<<<slots, kThreads, 0, st>>>(a, part_loss, off, pix1_dev, pix2_dev, mask1_dev, mask2_dev);
  final_kernel<<<1, kThreads, 0, st>>>(a, part_loss, reduction, out_dev);
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}
