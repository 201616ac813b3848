// Streaming variant of the fused global-alignment step (sm_90a): persistent grid, every WARP is an independent
// pipeline over its own list of work items.
//
// Same mathematics and the same HBM traffic as csrc/align_step.cu (32*E*P + 24*n*P bytes per iteration, SURVEY §8d;
// reference: dust3r/cloud_opt/optimizer.py:188-201, base_opt.py:246-273,352-366) -- what changes is how the SM is fed:
//
//   * work item = <= PPT slots of 64 consecutive pixels of one image; persistent warp w owns a contiguous list of
//     items (host-balanced to within one slot), so there are no waves, no per-CTA set-up and no tail;
//   * each warp runs a private NST-deep shared-memory ring filled by cp.async.bulk (lane 0 issues, mbarrier
//     tx-count completes).  The stage sequence of an item is   L | E_0 .. E_{deg-1} | MV :
//        L   item header (host-built constants) + the image's transform row + the item's log-depths,
//        E_k the entry's transform row (-M, -t) + the entry's observations for the item's pixels,
//        MV  the image's transform row + log-depth, exp_avg, exp_avg_sq slices for the in-place Adam update;
//     no warp ever waits for another warp: the ring is refilled by the warp that drained it, across item boundaries;
//   * observations are stored slot-interleaved as pixel PAIRS, [32 x (xA,xB,yA,yB)] [32 x (zA,zB,wA,wB)] per slot, so
//     two LDS.128 hand the thread two pixels as packed pairs and the whole residual / gradient algebra runs on
//     pixel pairs (two independent dependency chains per thread);
//   * the 13 per-entry sums are reduced across the warp through a transpose in the just-drained stage buffer
//     (13 STS + 4 LDS.128 + 16 FADD instead of a 16-shuffle butterfly), accumulated per warp in shared memory over
//     all of the warp's items of an image, and leave the SM once per (warp, image) as 2^44 fixed-point integer
//     atomics (order independent -> bit-reproducible), exactly like the general kernel;
//   * sqrt / reciprocal / exp of the per-pixel Adam update and unprojection use the MUFU approximations (<= 2 ulp).
//
// The last CTA of the grid (ticket) runs the same small-parameter step as the general kernel (align_common.cuh).
#include "align_common.cuh"

namespace d3r {
namespace align {

constexpr int kSWarps = 8;
constexpr int kSThreads = kSWarps * 32;
constexpr int kHdrBytes = 128;      // stage header: item header (64) + image row (64) | entry row (48) | image row (64)
constexpr int kSlotBytes = 1024;    // 64 pixels x 16 bytes
constexpr int kScrStride = 36;      // floats per row of the transpose scratch (bank-conflict-free LDS.128 rows)

static_assert(sizeof(d3r_align_item) == 64, "d3r_align_item must be 64 bytes");

typedef unsigned long long f2;      // two packed fp32 (lo = pixel A, hi = pixel B)
__device__ __forceinline__ f2 pack2(float lo, float hi) { f2 d; asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "f"(lo), "f"(hi)); return d; }
__device__ __forceinline__ f2 bc2(float x) { return pack2(x, x); }
__device__ __forceinline__ void unpack2(f2 v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
// Hopper has no packed fp32 arithmetic: each pair operation is two scalar round-to-nearest operations, which gives
// the same bits per lane as a packed one
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(c, c0, c1);
  return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ f2 add2(f2 a, f2 b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1); unpack2(b, b0, b1);
  return pack2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ f2 mul2(f2 a, f2 b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1); unpack2(b, b0, b1);
  return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ float rsqrt_approx(float x) { float y; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sqrt_approx(float x) { float y; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sb_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void sb_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sb_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  uint32_t spins = 0;
  do {
    asm volatile(
        "{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    // a stage that never lands is a bug (byte count mismatch): fail the launch instead of hanging the GPU
    if (!done && ++spins > (1u << 22)) __trap();
  } while (!done);
}
__device__ __forceinline__ void sb_bulk(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// Streamed data (observations, log-depths, Adam moments) is loaded with the L2 evict_first policy: it is dead after one use
// within an iteration, and at default priority 200+ MB of it per iteration push everything else out of the 126 MB L2 --
// including the instructions and inputs of the small-parameter step, which one CTA then re-fetches from DRAM on the critical
// path.  Among themselves evict_first lines still age in order, so the reversed traversal of odd iterations keeps finding the
// tail of the previous pass.
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void sb_bulk_stream(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
}

struct ProdState {          // per warp, touched by lane 0 only
  int item, item_end;
  int phase, deg;           // stage to issue next: 0 = L, 1..deg = E_{phase-1}, deg+1 = MV
  int slot;                 // ring slot it goes to
  uint32_t px_bytes, pay_bytes;
  int slab_units;           // 16-byte units between the slabs of consecutive entries
  const float* row;         // transform row of the next entry
  const uint4* obs;         // observations of the next entry for this item's pixels
  const float* irow;        // image transform row
  int64_t pix0;             // first pixel of the item in logd / logd_m / logd_v
};

// Sums NV per-lane values over the warp through a transpose in shared memory.  Lanes 2v and 2v+1 return the total of
// value v (v < NV <= 16); `scr` needs NV * kScrStride floats, 16-byte aligned.
template <int NV>
__device__ __forceinline__ float warp_transpose_sum(const float (&a)[NV], float* scr, int lane) {
#pragma unroll
  for (int v = 0; v < NV; ++v) scr[v * kScrStride + lane] = a[v];
  __syncwarp();
  float t = 0.f;
  if (lane < 2 * NV) {
    const float4* row = reinterpret_cast<const float4*>(scr + (lane >> 1) * kScrStride + (lane & 1) * 16);
    const float4 p0 = row[0], p1 = row[1], p2 = row[2], p3 = row[3];
    t = (((p0.x + p0.y) + (p0.z + p0.w)) + ((p1.x + p1.y) + (p1.z + p1.w))) +
        (((p2.x + p2.y) + (p2.z + p2.w)) + ((p3.x + p3.y) + (p3.z + p3.w)));
  }
  t += __shfl_xor_sync(0xffffffffu, t, 1);
  return t;
}

// Issues the next stage of this warp's sequence into its ring slot (lane 0 only).
template <int PPT, int NST>
__device__ __forceinline__ void produce_next(const d3r_align_desc& D, const Workspace& ws, const d3r_align_item* item_tab,
                                             ProdState* ps, uint8_t* ring, uint64_t* full) {
  constexpr int kStage = kHdrBytes + PPT * kSlotBytes;
  const int item = ps->item;
  if (item >= ps->item_end) return;
  const int s = ps->slot;
  const uint32_t dst = s_u32(ring + s * kStage);
  const uint32_t bar = s_u32(&full[s]);
  const int phase = ps->phase;
  const uint64_t pol = policy_evict_first();
  ps->slot = (s + 1 == NST) ? 0 : s + 1;
  if (phase == 0) {                                  // L: header | image row | log-depth slice
    const d3r_align_item* gh = item_tab + item;
    const d3r_align_item h = *gh;
    const uint32_t px_bytes = uint32_t(h.npx) * 4u;
    const float* irow = ws.imgT + int64_t(h.img) * kImgT;
    sb_expect_tx(bar, 64u + 64u + px_bytes);
    sb_bulk(dst, gh, 64u, bar);
    sb_bulk(dst + 64u, irow, 64u, bar);
    sb_bulk_stream(dst + kHdrBytes, D.logd + h.pix0, px_bytes, bar, pol);
    ps->deg = h.deg; ps->px_bytes = px_bytes; ps->pay_bytes = uint32_t(h.nslots) * kSlotBytes; ps->slab_units = h.slab_units;
    ps->row = ws.entT + int64_t(h.e0) * kEdgeT;
    ps->obs = reinterpret_cast<const uint4*>(D.obs) + h.obs0;
    ps->irow = irow; ps->pix0 = h.pix0;
    ps->phase = 1;
  } else if (phase <= ps->deg) {                     // E_k: entry row | observations
    const float* row = ps->row;
    const uint4* obs = ps->obs;
    const uint32_t pay = ps->pay_bytes;
    sb_expect_tx(bar, 48u + pay);
    sb_bulk(dst, row, 48u, bar);
    sb_bulk_stream(dst + kHdrBytes, obs, pay, bar, pol);
    ps->row = row + kEdgeT;
    ps->obs = obs + ps->slab_units;
    ps->phase = phase + 1;
  } else {                                           // MV: image row | log-depth | exp_avg | exp_avg_sq
    const uint32_t px_bytes = ps->px_bytes;
    const int64_t pix0 = ps->pix0;
    sb_expect_tx(bar, 64u + 3u * px_bytes);
    sb_bulk(dst, ps->irow, 64u, bar);
    sb_bulk_stream(dst + kHdrBytes, D.logd + pix0, px_bytes, bar, pol);
    sb_bulk_stream(dst + kHdrBytes + PPT * 256, D.logd_m + pix0, px_bytes, bar, pol);
    sb_bulk_stream(dst + kHdrBytes + 2 * PPT * 256, D.logd_v + pix0, px_bytes, bar, pol);
    ps->item = item + 1;
    ps->phase = 0;
  }
}

// ---- per-stage math, specialised on the number of slots of the item so that the slots' instruction streams are
// ---- straight-line code the scheduler can interleave (no per-slot branches)
template <int NS, int PPT>
__device__ __forceinline__ void unproject_slots(const uint8_t* slot, int lane, int npx, f2 (&X)[PPT][3], f2 (&G)[PPT][3]) {
  const d3r_align_item* h = reinterpret_cast<const d3r_align_item*>(slot);
  const int W = h->W, u0 = h->u0, v0 = h->v0;
  const float invW = h->inv_w;
  const float4* ir = reinterpret_cast<const float4*>(slot + 64);
  const float4 i0 = ir[0], i1 = ir[1], i2 = ir[2], i3 = ir[3];   // R0..R3 | R4..R7 | R8 T0 T1 T2 | ifx ify cx cy
  const float2* ldp = reinterpret_cast<const float2*>(slot + kHdrBytes);
#pragma unroll
  for (int kk = 0; kk < PPT; ++kk) {
    if (kk < NS) {
      const int j = kk * 32 + lane;
      float2 ld = make_float2(0.f, 0.f);
      if (2 * j < npx) ld = ldp[j];
      const f2 d = pack2(__expf(ld.x), __expf(ld.y));
      const int a = u0 + 2 * j;
      const int dv = __float2int_rz((float(a) + 0.5f) * invW);
      const int uA = a - dv * W, vA = v0 + dv;
      int uB = uA + 1, vB = vA;
      if (uB == W) { uB = 0; vB = vA + 1; }
      // c0 = d * (u - cx) / fx, c1 = d * (v - cy) / fy   (optimizer.py:203-211)
      const f2 c0 = mul2(mul2(d, add2(pack2(float(uA), float(uB)), bc2(-i3.z))), bc2(i3.x));
      const f2 c1 = mul2(mul2(d, add2(pack2(float(vA), float(vB)), bc2(-i3.w))), bc2(i3.y));
      X[kk][0] = fma2(bc2(i0.x), c0, fma2(bc2(i0.y), c1, fma2(bc2(i0.z), d, bc2(i2.y))));
      X[kk][1] = fma2(bc2(i0.w), c0, fma2(bc2(i1.x), c1, fma2(bc2(i1.y), d, bc2(i2.z))));
      X[kk][2] = fma2(bc2(i1.z), c0, fma2(bc2(i1.w), c1, fma2(bc2(i2.x), d, bc2(i2.w))));
    } else {
      X[kk][0] = X[kk][1] = X[kk][2] = 0ull;
    }
    G[kk][0] = G[kk][1] = G[kk][2] = 0ull;
  }
}

template <bool kL2, int NS, int PPT>
__device__ __forceinline__ void entry_slots(const uint8_t* slot, int lane, const f2 (&X)[PPT][3], f2 (&G)[PPT][3],
                                            float (&a13)[kEntVals]) {
  const float4* er = reinterpret_cast<const float4*>(slot);
  const float4 m0 = er[0], m1 = er[1], m2 = er[2];    // -M0..-M3 | -M4..-M7 | -M8 -t0 -t1 -t2
  const uint8_t* pay = slot + kHdrBytes + lane * 16;
  f2 acc[kEntVals];
#pragma unroll
  for (int v = 0; v < kEntVals; ++v) acc[v] = 0ull;
#pragma unroll
  for (int kk = 0; kk < NS; ++kk) {
    const ulonglong2 p0 = *reinterpret_cast<const ulonglong2*>(pay + kk * kSlotBytes);
    const ulonglong2 p1 = *reinterpret_cast<const ulonglong2*>(pay + kk * kSlotBytes + 512);
    const f2 qx = p0.x, qy = p0.y, qz = p1.x, w = p1.y;
    // r = X - (M q + t)
    const f2 r0 = fma2(bc2(m0.x), qx, fma2(bc2(m0.y), qy, fma2(bc2(m0.z), qz, add2(X[kk][0], bc2(m2.y)))));
    const f2 r1 = fma2(bc2(m0.w), qx, fma2(bc2(m1.x), qy, fma2(bc2(m1.y), qz, add2(X[kk][1], bc2(m2.z)))));
    const f2 r2 = fma2(bc2(m1.z), qx, fma2(bc2(m1.w), qy, fma2(bc2(m2.x), qz, add2(X[kk][2], bc2(m2.w)))));
    const f2 rho2 = fma2(r0, r0, fma2(r1, r1, mul2(r2, r2)));
    f2 gs;
    if (kL2) {
      acc[12] = fma2(w, rho2, acc[12]);
      gs = add2(w, w);
    } else {
      // torch's norm backward yields 0 at ||r|| == 0: r == 0 there, so a finite 1/||r|| stand-in gives g = 0
      float ra, rb;
      unpack2(rho2, ra, rb);
      const f2 inv = pack2(rsqrt_approx(fmaxf(ra, 1e-36f)), rsqrt_approx(fmaxf(rb, 1e-36f)));
      acc[12] = fma2(w, mul2(rho2, inv), acc[12]);
      gs = mul2(w, inv);
    }
    const f2 g0 = mul2(gs, r0), g1 = mul2(gs, r1), g2 = mul2(gs, r2);
    G[kk][0] = add2(G[kk][0], g0); G[kk][1] = add2(G[kk][1], g1); G[kk][2] = add2(G[kk][2], g2);
    acc[0] = fma2(g0, qx, acc[0]); acc[1] = fma2(g0, qy, acc[1]); acc[2] = fma2(g0, qz, acc[2]);
    acc[3] = fma2(g1, qx, acc[3]); acc[4] = fma2(g1, qy, acc[4]); acc[5] = fma2(g1, qz, acc[5]);
    acc[6] = fma2(g2, qx, acc[6]); acc[7] = fma2(g2, qy, acc[7]); acc[8] = fma2(g2, qz, acc[8]);
    acc[9] = add2(acc[9], g0); acc[10] = add2(acc[10], g1); acc[11] = add2(acc[11], g2);
  }
#pragma unroll
  for (int v = 0; v < kEntVals; ++v) { float lo, hi; unpack2(acc[v], lo, hi); a13[v] = lo + hi; }
}

template <int NS, int PPT>
__device__ __forceinline__ void adam_slots(const d3r_align_desc& D, const uint8_t* slot, int lane, int npx, int64_t pix0,
                                           float step_size, float inv_bc2s, const f2 (&X)[PPT][3], const f2 (&G)[PPT][3],
                                           float (&s12)[kImgVals]) {
  const float4 i2 = reinterpret_cast<const float4*>(slot)[2];   // R8 T0 T1 T2
  const float2* ldp = reinterpret_cast<const float2*>(slot + kHdrBytes);
  const float2* mp = reinterpret_cast<const float2*>(slot + kHdrBytes + PPT * 256);
  const float2* vp = reinterpret_cast<const float2*>(slot + kHdrBytes + 2 * PPT * 256);
  f2 S[kImgVals];
#pragma unroll
  for (int v = 0; v < kImgVals; ++v) S[v] = 0ull;
#pragma unroll
  for (int kk = 0; kk < NS; ++kk) {
    const int j = kk * 32 + lane;
    if (2 * j < npx) {
      // Y = X - T = R c ; dX/dlogd = Y (c is linear in the depth)
      const f2 y0 = add2(X[kk][0], bc2(-i2.y)), y1 = add2(X[kk][1], bc2(-i2.z)), y2 = add2(X[kk][2], bc2(-i2.w));
      const f2 gd = fma2(G[kk][0], y0, fma2(G[kk][1], y1, mul2(G[kk][2], y2)));
      S[0] = fma2(G[kk][0], y0, S[0]); S[1] = fma2(G[kk][0], y1, S[1]); S[2] = fma2(G[kk][0], y2, S[2]);
      S[3] = fma2(G[kk][1], y0, S[3]); S[4] = fma2(G[kk][1], y1, S[4]); S[5] = fma2(G[kk][1], y2, S[5]);
      S[6] = fma2(G[kk][2], y0, S[6]); S[7] = fma2(G[kk][2], y1, S[7]); S[8] = fma2(G[kk][2], y2, S[8]);
      S[9] = add2(S[9], G[kk][0]); S[10] = add2(S[10], G[kk][1]); S[11] = add2(S[11], G[kk][2]);
      const float2 ld = ldp[j], mm = mp[j], vv = vp[j];
      // torch.optim.Adam: m += (1-b1)(g-m); v = v*b2 + (1-b2) g g; p -= step * m / (sqrt(v)/sqrt(bc2) + eps)
      const f2 m_old = pack2(mm.x, mm.y);
      const f2 m_new = fma2(bc2(1.f - D.beta1), fma2(bc2(-1.f), m_old, gd), m_old);
      const f2 v_new = fma2(mul2(bc2(1.f - D.beta2), gd), gd, mul2(pack2(vv.x, vv.y), bc2(D.beta2)));
      float va, vb;
      unpack2(v_new, va, vb);
      const f2 denom = fma2(pack2(sqrt_approx(va), sqrt_approx(vb)), bc2(inv_bc2s), bc2(D.adam_eps));
      float da, db;
      unpack2(denom, da, db);
      const f2 upd = mul2(m_new, pack2(rcp_approx(da), rcp_approx(db)));
      const f2 ld_new = fma2(bc2(-step_size), upd, pack2(ld.x, ld.y));
      reinterpret_cast<f2*>(D.logd + pix0)[j] = ld_new;
      reinterpret_cast<f2*>(D.logd_m + pix0)[j] = m_new;
      reinterpret_cast<f2*>(D.logd_v + pix0)[j] = v_new;
    }
  }
#pragma unroll
  for (int v = 0; v < kImgVals; ++v) { float lo, hi; unpack2(S[v], lo, hi); s12[v] = lo + hi; }
}

template <bool kL2, int PPT, int NST>
__global__ void __launch_bounds__(kSThreads, 2)
align_stream_kernel(const __grid_constant__ d3r_align_desc D, int it) {
  static_assert(PPT == 3, "the per-slot specialisations below are written for 3 slots per item");
  constexpr int kStage = kHdrBytes + PPT * kSlotBytes;
  extern __shared__ __align__(128) uint8_t s_dyn[];
  __shared__ __align__(8) uint64_t s_full[kSWarps][NST];
  __shared__ __align__(16) ProdState s_prod[kSWarps];
  __shared__ float s_red[40];
  __shared__ int s_flag;

  const Workspace ws = carve(D.workspace, D.n_imgs, D.n_edges);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gw = blockIdx.x * kSWarps + warp;
  const int Wn = D.stream_window;
  const int acc_floats = (Wn * kEntVals + 16 + 31) & ~31;
  const size_t per_warp = size_t(NST) * kStage + size_t(acc_floats) * 4;
  uint8_t* ring = s_dyn + warp * per_warp;
  float* s_acc = reinterpret_cast<float*>(ring + NST * kStage);   // [Wn][13] entry sums of the open window
  float* s_img = s_acc + Wn * kEntVals;                           // [12] image sums
  uint64_t* full = s_full[warp];
  ProdState* ps = &s_prod[warp];

  // odd iterations walk the reversed item table when the host provides one (L2 reuse across iterations)
  const bool rev = (it & 1) && D.items_rev != nullptr;
  const int32_t* wip = rev ? D.warp_item_ptr_rev : D.warp_item_ptr;
  const d3r_align_item* item_tab = reinterpret_cast<const d3r_align_item*>(rev ? D.items_rev : D.items);
  const int ib = wip[gw], ie = wip[gw + 1];
  unsigned long long* dbg = g_align_dbg ? g_align_dbg + 4 * size_t(gw) : nullptr;   // per-warp timeline (debug aid)
  if (dbg && lane == 0) dbg[0] = gtime();
  if (lane == 0) {
    for (int s = 0; s < NST; ++s) sb_init(s_u32(&full[s]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    ps->item = ib; ps->item_end = ie; ps->phase = 0; ps->slot = 0;
  }
  for (int i = lane; i < Wn * kEntVals + 16; i += 32) s_acc[i] = 0.f;
  __syncwarp();

  // everything below reads what the previous iteration wrote (transforms, log-depths, Adam moments)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (dbg && lane == 0) dbg[1] = gtime();
  if (lane == 0)
    for (int s = 0; s < NST; ++s) produce_next<PPT, NST>(D, ws, item_tab, ps, ring, full);
  __syncwarp();

  const float step_size = D.sched[it * 4 + 1];
  const float inv_bc2s = 1.f / D.sched[it * 4 + 2];
  const bool train = !D.eval_only;

  int si = 0;                           // ring slot of the next stage to consume
  uint32_t par = 0;                     // its mbarrier phase parity
  auto advance = [&]() { if (++si == NST) { si = 0; par ^= 1u; } };
  int acc_e0 = 0, acc_cnt = 0, acc_img = -1;               // open entry window of s_acc: entries [acc_e0, acc_e0 + acc_cnt)
  int simg = -1;                                           // image of s_img

  auto flush_entries = [&]() {
    if (acc_cnt > 0) {
      for (int idx = lane; idx < acc_cnt * kEntVals; idx += 32) {
        const float v = s_acc[idx];
        s_acc[idx] = 0.f;
        fix_add(ws.ent_acc + int64_t(acc_e0) * kEntVals + idx, v, ws.flags);
      }
      __syncwarp();
    }
    acc_cnt = 0;
  };
  auto flush_image = [&]() {
    if (simg >= 0 && lane < kImgVals) {
      fix_add(ws.img_acc + int64_t(simg) * kImgVals + lane, s_img[lane], ws.flags);
      s_img[lane] = 0.f;
    }
    __syncwarp();
    simg = -1;
  };

  for (int item = ib; item < ie; ++item) {
    // ------------------------------------------------------------------ L stage: unproject this item's pixels
    uint8_t* slot = ring + si * kStage;
    sb_wait(s_u32(&full[si]), par);
    const d3r_align_item* h = reinterpret_cast<const d3r_align_item*>(slot);
    const int img = h->img, nslots = h->nslots, npx = h->npx, e0 = h->e0, deg = h->deg;
    const int64_t pix0 = h->pix0;
    f2 X[PPT][3], G[PPT][3];
    if (nslots == 3) unproject_slots<3, PPT>(slot, lane, npx, X, G);
    else if (nslots == 2) unproject_slots<2, PPT>(slot, lane, npx, X, G);
    else unproject_slots<1, PPT>(slot, lane, npx, X, G);
    __syncwarp();
    if (lane == 0) produce_next<PPT, NST>(D, ws, item_tab, ps, ring, full);
    advance();

    if (simg != img) { flush_image(); simg = img; }
    // a window that holds ALL entries of the image stays open across the warp's items of that image
    if (acc_img != img || acc_e0 != e0 || acc_cnt == 0) {
      flush_entries();
      acc_img = img; acc_e0 = e0; acc_cnt = min(Wn, deg);
    }

    // ------------------------------------------------------------------ E stages: residuals against every entry
    int kin = 0;                          // index of entry k inside the open window
    for (int k = 0; k < deg; ++k, ++kin) {
      if (kin == Wn) {                    // more entries than the window holds: spill and open the next window
        flush_entries();
        acc_e0 = e0 + k; acc_cnt = min(Wn, deg - k); kin = 0;
      }
      slot = ring + si * kStage;
      sb_wait(s_u32(&full[si]), par);
      float a13[kEntVals];
      if (nslots == 3) entry_slots<kL2, 3, PPT>(slot, lane, X, G, a13);
      else if (nslots == 2) entry_slots<kL2, 2, PPT>(slot, lane, X, G, a13);
      else entry_slots<kL2, 1, PPT>(slot, lane, X, G, a13);
      __syncwarp();                               // every lane is done reading the observations of this stage
      const float tot = warp_transpose_sum<kEntVals>(a13, reinterpret_cast<float*>(slot + kHdrBytes), lane);
      if (!(lane & 1) && lane < 2 * kEntVals) s_acc[kin * kEntVals + (lane >> 1)] += tot;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) produce_next<PPT, NST>(D, ws, item_tab, ps, ring, full);
      advance();
    }

    // ------------------------------------------------------------------ MV stage: depth gradient + Adam in place
    slot = ring + si * kStage;
    sb_wait(s_u32(&full[si]), par);
    if (train) {
      float s12[kImgVals];
      if (nslots == 3) adam_slots<3, PPT>(D, slot, lane, npx, pix0, step_size, inv_bc2s, X, G, s12);
      else if (nslots == 2) adam_slots<2, PPT>(D, slot, lane, npx, pix0, step_size, inv_bc2s, X, G, s12);
      else adam_slots<1, PPT>(D, slot, lane, npx, pix0, step_size, inv_bc2s, X, G, s12);
      __syncwarp();
      const float tot = warp_transpose_sum<kImgVals>(s12, reinterpret_cast<float*>(slot + kHdrBytes), lane);
      if (!(lane & 1) && lane < 2 * kImgVals) s_img[lane >> 1] += tot;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncwarp();
    if (lane == 0) produce_next<PPT, NST>(D, ws, item_tab, ps, ring, full);
    advance();
    if (deg > Wn) flush_entries();        // a spilled image starts its next item from window 0 again
  }
  flush_entries();
  flush_image();
  if (dbg && lane == 0) dbg[2] = gtime();
  const int scr_floats = int(size_t(kSWarps) * per_warp / 4);
  if (warp == 0) prefetch_small_step_inputs(D, ws, it, scr_floats, lane, 32);

  // ---- grid ticket: the last CTA to finish runs the small-parameter step ----
  __syncthreads();
  if (tid == 0) s_flag = (grid_ticket(D.counters) == int(gridDim.x) - 1);
  __syncthreads();
  if (dbg && lane == 0) dbg[3] = gtime();
  if (!s_flag) return;
  if (tid == 0) D.counters[0] = 0;   // re-arm for the next launch
  // every stage this CTA issued has been consumed: the ring is idle and serves as the small step's scratch
  small_step(D, ws, it, s_red, reinterpret_cast<float*>(s_dyn), scr_floats);
  D3R_TSTAMP(5);
}

// ---- one launch packs every entry (device-resident forward output -> observation layout) ----------------------
__device__ __forceinline__ float conf_trf(float c, int mode) {
  switch (mode) {
    case D3R_CONF_LOG: return logf(c);
    case D3R_CONF_SQRT: return sqrtf(c);
    case D3R_CONF_M1: return c - 1.f;
    default: return c;
  }
}

__global__ void __launch_bounds__(256) pack_entries_kernel(const d3r_pack_entry* __restrict__ table, int conf_mode,
                                                           int stream_layout, float4* __restrict__ obs) {
  const d3r_pack_entry e = table[blockIdx.y];
  float4* out = obs + e.obs_off;
  if (!stream_layout) {
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < e.area; p += gridDim.x * blockDim.x)
      out[p] = make_float4(e.pts[int64_t(p) * 3 + 0], e.pts[int64_t(p) * 3 + 1], e.pts[int64_t(p) * 3 + 2], conf_trf(e.conf[p], conf_mode));
    return;
  }
  // one thread per pixel pair; slot = 32 pairs = [32 x (xA,xB,yA,yB)] [32 x (zA,zB,wA,wB)]
  const int npairs_padded = ((e.area + 63) / 64) * 32;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < npairs_padded; j += gridDim.x * blockDim.x) {
    const int pA = 2 * j, pB = 2 * j + 1;
    float xa = 0.f, ya = 0.f, za = 0.f, wa = 0.f, xb = 0.f, yb = 0.f, zb = 0.f, wb = 0.f;
    if (pA < e.area) {
      xa = e.pts[int64_t(pA) * 3 + 0]; ya = e.pts[int64_t(pA) * 3 + 1]; za = e.pts[int64_t(pA) * 3 + 2];
      wa = e.coef * conf_trf(e.conf[pA], conf_mode);
    }
    if (pB < e.area) {
      xb = e.pts[int64_t(pB) * 3 + 0]; yb = e.pts[int64_t(pB) * 3 + 1]; zb = e.pts[int64_t(pB) * 3 + 2];
      wb = e.coef * conf_trf(e.conf[pB], conf_mode);
    }
    float4* slot = out + int64_t(j >> 5) * 64;
    slot[j & 31] = make_float4(xa, xb, ya, yb);
    slot[32 + (j & 31)] = make_float4(za, zb, wa, wb);
  }
}

// world points for the streaming layout's owners are produced by the general pts3d kernel (layout independent)

template <bool kL2, int PPT, int NST>
static int launch_stream_t(const d3r_align_desc* desc, int it_begin, int it_end, cudaStream_t st) {
  constexpr int kStage = kHdrBytes + PPT * kSlotBytes;
  const int acc_floats = (desc->stream_window * kEntVals + 16 + 31) & ~31;
  const size_t smem = size_t(kSWarps) * (size_t(NST) * kStage + size_t(acc_floats) * 4);
  // per device: the opt-in is a per-context function attribute (a process may drive several GPUs)
  D3R_CUDA(cudaFuncSetAttribute(align_stream_kernel<kL2, PPT, NST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  D3R_CUDA(cudaFuncSetAttribute(align_stream_kernel<kL2, PPT, NST>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)desc->stream_grid);
  cfg.blockDim = dim3(kSThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  for (int it = it_begin; it < it_end; ++it) D3R_CUDA(cudaLaunchKernelEx(&cfg, align_stream_kernel<kL2, PPT, NST>, *desc, it));
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}

int stream_set_debug(unsigned long long* p) {   // this translation unit's copy of the timeline pointer
  D3R_CUDA(cudaMemcpyToSymbol(g_align_dbg, &p, sizeof(p)));
  return D3R_OK;
}

size_t stream_smem_bytes(int ppt, int nst, int window) {
  const int acc_floats = (window * kEntVals + 16 + 31) & ~31;
  return size_t(kSWarps) * (size_t(nst) * (kHdrBytes + ppt * kSlotBytes) + size_t(acc_floats) * 4);
}

int launch_stream(const d3r_align_desc* desc, int it_begin, int it_end, cudaStream_t st) {
  D3R_CHECK_ARG(desc->items && desc->warp_item_ptr && desc->n_items > 0 && desc->stream_grid > 0,
                "d3r_align_run: streaming kernel selected without a work-item table");
  D3R_CHECK_ARG(desc->stream_ppt == 3, "d3r_align_run: stream_ppt=%d is not built (3)", desc->stream_ppt);
  D3R_CHECK_ARG(desc->stream_window >= 1, "d3r_align_run: stream_window must be >= 1");
  // ring depth: 4 stages while the entry window leaves room for two CTAs per SM, else 3
  const size_t budget = 113 * 1024;
  const bool deep = stream_smem_bytes(3, 4, desc->stream_window) <= budget;
  D3R_CHECK_ARG(deep || stream_smem_bytes(3, 3, desc->stream_window) <= budget, "d3r_align_run: stream_window=%d does not fit shared memory",
                desc->stream_window);
  if (desc->dist_l2) return deep ? launch_stream_t<true, 3, 4>(desc, it_begin, it_end, st) : launch_stream_t<true, 3, 3>(desc, it_begin, it_end, st);
  return deep ? launch_stream_t<false, 3, 4>(desc, it_begin, it_end, st) : launch_stream_t<false, 3, 3>(desc, it_begin, it_end, st);
}

}  // namespace align
}  // namespace d3r

using namespace d3r;
using namespace d3r::align;

extern "C" int d3r_sizeof_align_item(void) { return (int)sizeof(d3r_align_item); }
extern "C" int d3r_sizeof_pack_entry(void) { return (int)sizeof(d3r_pack_entry); }
extern "C" int d3r_align_stream_slots_per_item(void) { return 3; }
extern "C" int d3r_align_stream_warps_per_cta(void) { return kSWarps; }
/* largest entry window (entries whose sums a warp keeps in shared memory) that still allows two CTAs per SM */
extern "C" int d3r_align_stream_max_window(void) {
  int w = 1;
  while (stream_smem_bytes(3, 3, w + 1) <= 113 * 1024) ++w;
  return w;
}

extern "C" int d3r_align_pack_entries(const d3r_pack_entry* table_dev, int32_t n_entries, int32_t max_area, int32_t conf_mode,
                                      int32_t stream_layout, void* obs_dev, void* stream) {
  D3R_CHECK_ARG(table_dev && obs_dev && n_entries > 0 && max_area > 0, "d3r_align_pack_entries: bad arguments");
  D3R_CHECK_ARG(conf_mode >= D3R_CONF_ID && conf_mode <= D3R_CONF_M1, "d3r_align_pack_entries: bad conf_mode %d", conf_mode);
  D3R_CHECK_ARG(n_entries <= 65535, "d3r_align_pack_entries: too many entries (%d) for one launch", n_entries);
  const int work = stream_layout ? ((max_area + 63) / 64) * 32 : max_area;
  const int bx = (work + 255) / 256 < 1024 ? (work + 255) / 256 : 1024;
  prof::Scope scope("align_pack", (cudaStream_t)stream, 0.0, 0.0, 1);
  pack_entries_kernel<<<dim3((unsigned)bx, (unsigned)n_entries), 256, 0, (cudaStream_t)stream>>>(table_dev, conf_mode, stream_layout,
                                                                                               reinterpret_cast<float4*>(obs_dev));
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}
