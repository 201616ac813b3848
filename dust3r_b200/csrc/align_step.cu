// Fused global-alignment step for H100 (sm_90a): one launch per Adam iteration.
//
// Replaces, per iteration, the ~dozens of elementwise/bmm/gather kernels + autograd + foreach-Adam
// of the reference loop (dust3r/cloud_opt/base_opt.py:352-366 driving optimizer.py:188-201 or
// base_opt.py:246-273).  HBM-bound fp32: every observation float4 (pred.xyz, weight) is read once,
// every log-depth and its two Adam moments are read and written once  -> 32*E*P + 24*n*P bytes
// per iteration (SURVEY §8d).  No tensor cores (K=3 contractions).
//
// Work decomposition
//   CTA  = (image i, chunk of kChunk pixels).  Each thread owns kPPT pixels, keeps their world
//          points X and the accumulated dL/dX in registers and loops over the entries
//          (edge, side) incident to image i, streaming the entry's float4 observations.
//   per entry the CTA reduces 13 sums (sum g (x) q, sum g, loss) with warp shuffles -> smem ->
//          one partial row in global memory (deterministic: no float atomics anywhere).
//   after the entry loop the thread has dL/dX for its pixels: depth gradient + Adam in place.
//   last CTA of an image (atomic ticket) reduces that image's partial rows; last CTA of the grid
//          turns the sums into pose/focal/pp/pairwise-pose gradients (quaternion-normalise,
//          signed_expm1 and the mean-coupled scale backward done analytically), applies Adam and
//          writes the transforms of the next iteration.
#include "align_common.cuh"

namespace d3r {
namespace align {

__global__ void __launch_bounds__(kThreads) prepare_kernel(const __grid_constant__ d3r_align_desc D) {
  __shared__ float s_red[40];
  Workspace ws = carve(D.workspace, D.n_imgs, D.n_edges);
  compute_transforms(D, ws, s_red);
}


// ---- the per-iteration kernel ---------------------------------------------------------------
// 8 warps, all computing; lane 0 of warp 0 doubles as the producer: each incident entry's float4 observations
// for this CTA's pixel chunk are streamed into a 3-stage shared-memory ring with cp.async.bulk (TMA 1-D copies,
// mbarrier completion), refilled as soon as a stage is drained, so up to 2 x 84 KB of reads are in flight per
// SM independent of the warps' compute progress.
constexpr int kStages = 3;
constexpr int kEntTile = 16;               // entries whose per-warp partial sums are staged in smem at a time
constexpr int kRedVals = 16;               // 13 padded to 16 for the halving butterfly
using ptx::smem_u32;

// Sum 16 per-lane values across the warp with 16 shuffles (instead of 16 x 5): at every halving step a lane
// keeps one half of its values and trades the other half with its partner.  On return lane l holds the
// warp-wide total of value index (l >> 1) & 15 in v[0].
__device__ __forceinline__ float butterfly16(float (&v)[kRedVals], int lane) {
  {
    const bool up = lane & 16;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float send = up ? v[i] : v[i + 8];
      const float keep = up ? v[i + 8] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
  }
  {
    const bool up = lane & 8;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float send = up ? v[i] : v[i + 4];
      const float keep = up ? v[i + 4] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
  }
  {
    const bool up = lane & 4;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float send = up ? v[i] : v[i + 2];
      const float keep = up ? v[i + 2] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
  }
  {
    const bool up = lane & 2;
    const float send = up ? v[0] : v[1];
    const float keep = up ? v[1] : v[0];
    v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
  return v[0];
}

// Body of both instantiation families: kGrad = false is the training iteration (align_iter_kernel), kGrad = true the
// gradient export (align_grad_kernel): the depth stage writes dL/dlog-depth to go.logd_grad instead of running Adam, and
// the last CTA runs small_grad_step.
template <bool kGrad, bool kL2, int PPT>
__device__ __forceinline__ void iter_body(const d3r_align_desc& D, int it, const GradOut& go) {
  constexpr int kSlots = PPT * kThreads;     // pixel slots of this instantiation (>= chunk_px)
  extern __shared__ __align__(128) uint8_t s_dyn[];
  float4* s_obs = reinterpret_cast<float4*>(s_dyn);                                   // [kStages][kSlots]
  float* s_ent = reinterpret_cast<float*>(s_dyn + kStages * kSlots * sizeof(float4));  // [kEntTile][kWarps][13]
  __shared__ float s_img[kWarps * kImgVals];
  __shared__ float s_red[40];
  __shared__ int s_flag;
  __shared__ __align__(8) uint64_t s_full[kStages], s_empty[kStages];

  const Workspace ws = carve(D.workspace, D.n_imgs, D.n_edges);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int chunk = blockIdx.x;
  unsigned long long* dbg = g_align_dbg ? g_align_dbg + 4 * size_t(chunk) : nullptr;
  if (dbg && tid == 0) dbg[0] = gtime();
  const int img = D.chunk_img[chunk];
  const int lc = chunk - D.img_chunk_ptr[img];
  const int H = D.img_hw[img * 2 + 0], W = D.img_hw[img * 2 + 1];
  const int P = H * W;
  const int pbase = lc * D.chunk_px;                       // first pixel of this CTA
  const int npx = min(D.chunk_px, P - pbase);              // 1 .. kSlots
  const int64_t poff = D.img_pix_off[img];
  const int e0 = D.img_ent_ptr[img], e1 = D.img_ent_ptr[img + 1];
  const int deg = e1 - e0;
  const float4* obs_base = reinterpret_cast<const float4*>(D.obs);

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(smem_u32(&s_full[s]), 1);
      ptx::mbar_init(smem_u32(&s_empty[s]), kWarps);
    }
    ptx::fence_barrier_init();
  }
  // slots past the chunk are never written by the bulk copies: zero them once (weight 0 -> no contribution)
  for (int s = 0; s < kStages; ++s)
    for (int q = npx + tid; q < kSlots; q += kThreads) s_obs[s * kSlots + q] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();

  const uint32_t stage_bytes = uint32_t(npx) * 16u;
  auto produce = [&](int k) {   // called by one thread
    const int s = k % kStages;
    ptx::mbar_wait(smem_u32(&s_empty[s]), ((k / kStages) & 1) ^ 1);
    ptx::mbar_arrive_expect_tx(smem_u32(&s_full[s]), stage_bytes);
    ptx::bulk_g2s(smem_u32(s_obs + s * kSlots), obs_base + D.ent_obs_off[e0 + k] + pbase, stage_bytes, smem_u32(&s_full[s]));
  };
  if (tid == 0)
    for (int k = 0; k < min(kStages, deg); ++k) produce(k);

  // Programmatic dependent launch: everything above touches only per-problem constants (index tables, the
  // observation slabs) -- this iteration's CTAs were allowed to start it while the previous iteration's last CTA
  // was still in its small-parameter step.  Everything below reads what that step (and the previous depth update)
  // wrote, so wait here for the previous grid to complete and flush, and allow the NEXT iteration's CTAs to be
  // scheduled as soon as every CTA of this grid has got this far: they take the slots of this grid's last wave as its
  // CTAs retire, and block at their own wait.
  pdl::sync_with_predecessor();
  const float* iT = ws.imgT + img * kImgT;
  float R[9], T[3];
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = iT[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) T[k] = iT[9 + k];
  const float ifx = iT[12], ify = iT[13], cx = iT[14], cy = iT[15];

  float X[PPT][3], G[PPT][3];
#pragma unroll
  for (int k = 0; k < PPT; ++k) {
    const int q = tid + k * kThreads;
    const int p = pbase + q;
    const float ld = (q < npx) ? D.logd[poff + p] : 0.f;
    const float d = expf(ld);
    const int v = p / W, u = p - v * W;
    const float c0 = d * (float(u) - cx) * ifx, c1 = d * (float(v) - cy) * ify;
    X[k][0] = R[0] * c0 + R[1] * c1 + R[2] * d + T[0];
    X[k][1] = R[3] * c0 + R[4] * c1 + R[5] * d + T[1];
    X[k][2] = R[6] * c0 + R[7] * c1 + R[8] * d + T[2];
    G[k][0] = G[k][1] = G[k][2] = 0.f;
  }

  __shared__ __align__(16) float s_T[kEntTile][16];   // per-entry transform M (9), t (3), coef: staged per tile
  int stage = 0;
  uint32_t stage_phase = 0;
  for (int k0 = 0; k0 < deg; k0 += kEntTile) {
    const int kend = min(deg, k0 + kEntTile);
    // stage this tile's edge transforms in shared memory (one coalesced pass instead of 13 dependent LDGs per
    // entry per thread sitting on the critical path of every entry)
    if (tid < (kend - k0) * 13) {
      const int k = tid / 13, v = tid - k * 13;
      const int ent = e0 + k0 + k;
      s_T[k][v] = (v < 12) ? ws.edgeT[D.ent_edge[ent] * kEdgeT + v] : D.ent_coef[ent];
    }
    __syncthreads();
    for (int kk = k0; kk < kend; ++kk) {
      const float4 t0 = *reinterpret_cast<const float4*>(&s_T[kk - k0][0]);
      const float4 t1 = *reinterpret_cast<const float4*>(&s_T[kk - k0][4]);
      const float4 t2 = *reinterpret_cast<const float4*>(&s_T[kk - k0][8]);
      const float coef = s_T[kk - k0][12];
      const float M[9] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w, t2.x};
      const float t[3] = {t2.y, t2.z, t2.w};
      const int s = stage;
      ptx::mbar_wait(smem_u32(&s_full[s]), stage_phase);
      if (++stage == kStages) { stage = 0; stage_phase ^= 1; }
      const float4* so = s_obs + s * kSlots;
      float acc[kRedVals];
#pragma unroll
      for (int k = 0; k < kRedVals; ++k) acc[k] = 0.f;
#pragma unroll
      for (int k = 0; k < PPT; ++k) {
        const float4 o = so[tid + k * kThreads];
        const float qx = o.x, qy = o.y, qz = o.z;
        const float lw = coef * o.w;
        // r = X - (M q + t), written as FMA chains (the compiler may not re-associate fp32)
        const float r0 = X[k][0] - fmaf(M[0], qx, fmaf(M[1], qy, fmaf(M[2], qz, t[0])));
        const float r1 = X[k][1] - fmaf(M[3], qx, fmaf(M[4], qy, fmaf(M[5], qz, t[1])));
        const float r2 = X[k][2] - fmaf(M[6], qx, fmaf(M[7], qy, fmaf(M[8], qz, t[2])));
        const float rho2 = fmaf(r0, r0, fmaf(r1, r1, r2 * r2));
        float gs;
        if (kL2) {
          acc[12] = fmaf(lw, rho2, acc[12]);
          gs = 2.f * lw;
        } else {
          // torch's norm backward yields 0 at ||r|| == 0
          const float inv = rho2 > 0.f ? rsqrtf(rho2) : 0.f;
          acc[12] = fmaf(lw, rho2 * inv, acc[12]);
          gs = lw * inv;
        }
        const float g0 = gs * r0, g1 = gs * r1, g2 = gs * r2;
        G[k][0] += g0; G[k][1] += g1; G[k][2] += g2;
        acc[0] = fmaf(g0, qx, acc[0]); acc[1] = fmaf(g0, qy, acc[1]); acc[2] = fmaf(g0, qz, acc[2]);
        acc[3] = fmaf(g1, qx, acc[3]); acc[4] = fmaf(g1, qy, acc[4]); acc[5] = fmaf(g1, qz, acc[5]);
        acc[6] = fmaf(g2, qx, acc[6]); acc[7] = fmaf(g2, qy, acc[7]); acc[8] = fmaf(g2, qz, acc[8]);
        acc[9] += g0; acc[10] += g1; acc[11] += g2;
      }
      // this warp is done with the stage: hand it back, and (thread 0) refill it with entry kk + kStages
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(smem_u32(&s_empty[s]));
      if (tid == 0 && kk + kStages < deg) produce(kk + kStages);
      const float tot = butterfly16(acc, lane);
      const int vi = (lane >> 1) & 15;
      if (!(lane & 1) && vi < kEntVals) s_ent[((kk - k0) * kWarps + warp) * kEntVals + vi] = tot;
    }
    // cross-warp sums of this tile of entries (fixed order) -> deterministic fixed-point accumulation
    __syncthreads();
    for (int idx = tid; idx < (kend - k0) * kEntVals; idx += kThreads) {
      const int k = idx / kEntVals, v = idx - k * kEntVals;
      float sacc = 0.f;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) sacc += s_ent[(k * kWarps + w) * kEntVals + v];
      fix_add(ws.ent_acc + int64_t(e0 + k0 + k) * kEntVals + v, sacc, ws.flags);
    }
    __syncthreads();
  }

  // depth gradient + Adam (in place), per-image pose/focal sums
  float S[kRedVals];
#pragma unroll
  for (int k = 0; k < kRedVals; ++k) S[k] = 0.f;
  if (kGrad || !D.eval_only) {
    const float step_size = kGrad ? 0.f : D.sched[it * 4 + 1], bc2s = kGrad ? 1.f : D.sched[it * 4 + 2];
#pragma unroll
    for (int k = 0; k < PPT; ++k) {
      const int q = tid + k * kThreads;
      if (q < npx) {
        const int p = pbase + q;
        const float ld = D.logd[poff + p];
        const float d = expf(ld);
        const int v = p / W, u = p - v * W;
        const float c0 = d * (float(u) - cx) * ifx, c1 = d * (float(v) - cy) * ify;
        // dX/dlogd = R c  (c is linear in d)
        const float gd = G[k][0] * (X[k][0] - T[0]) + G[k][1] * (X[k][1] - T[1]) + G[k][2] * (X[k][2] - T[2]);
        if (kGrad) {
          go.logd_grad[poff + p] = gd;
        } else {
          float m = D.logd_m[poff + p], vv = D.logd_v[poff + p];
          const float nld = adam_update(ld, gd, m, vv, D.beta1, D.beta2, step_size, bc2s, D.adam_eps);
          D.logd[poff + p] = nld;
          D.logd_m[poff + p] = m;
          D.logd_v[poff + p] = vv;
        }
        S[0] += G[k][0] * c0; S[1] += G[k][0] * c1; S[2] += G[k][0] * d;
        S[3] += G[k][1] * c0; S[4] += G[k][1] * c1; S[5] += G[k][1] * d;
        S[6] += G[k][2] * c0; S[7] += G[k][2] * c1; S[8] += G[k][2] * d;
        S[9] += G[k][0]; S[10] += G[k][1]; S[11] += G[k][2];
      }
    }
  }
  {
    const float tot = butterfly16(S, lane);
    const int vi = (lane >> 1) & 15;
    if (!(lane & 1) && vi < kImgVals) s_img[warp * kImgVals + vi] = tot;
  }
  __syncthreads();
  if (tid < kImgVals) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) s += s_img[w * kImgVals + tid];
    fix_add(ws.img_acc + int64_t(img) * kImgVals + tid, s, ws.flags);
  }
  if (dbg && tid == 0) dbg[1] = gtime();

  if (!kGrad) prefetch_small_step_inputs(D, ws, it, int((size_t(kStages) * PPT * kThreads * sizeof(float4)) / 4), tid, kThreads);
  // ---- grid ticket: the last CTA to finish runs the small-parameter step ----
  __syncthreads();
  if (tid == 0) s_flag = (grid_ticket(D.counters) == int(gridDim.x) - 1);
  __syncthreads();
  if (!s_flag) {
    if (dbg && tid == 0) dbg[2] = gtime();
    return;
  }
  if (tid == 0) D.counters[0] = 0;   // re-arm for the next launch
  if (dbg && tid == 0) dbg[2] = gtime();
  if (kGrad)
    small_grad_step(D, ws, go, s_red);
  else
    small_step(D, ws, it, s_red, reinterpret_cast<float*>(s_dyn), int((size_t(kStages) * PPT * kThreads * sizeof(float4)) / 4));
  if (dbg && tid == 0) dbg[3] = gtime();
}

template <bool kL2, int PPT>
__global__ void __launch_bounds__(kThreads, 2)
align_iter_kernel(const __grid_constant__ d3r_align_desc D, int it) {
  iter_body<false, kL2, PPT>(D, it, GradOut{});
}

template <bool kL2, int PPT>
__global__ void __launch_bounds__(kThreads, 2)
align_grad_kernel(const __grid_constant__ d3r_align_desc D, GradOut go) {
  iter_body<true, kL2, PPT>(D, 0, go);
}

__global__ void __launch_bounds__(kThreads) pts3d_kernel(const __grid_constant__ d3r_align_desc D, float* out) {
  const Workspace ws = carve(D.workspace, D.n_imgs, D.n_edges);
  const int chunk = blockIdx.x;
  const int img = D.chunk_img[chunk];
  const int lc = chunk - D.img_chunk_ptr[img];
  const int H = D.img_hw[img * 2 + 0], W = D.img_hw[img * 2 + 1];
  const int P = H * W;
  const int64_t poff = D.img_pix_off[img];
  const float* iT = ws.imgT + img * kImgT;
  const int pend = min(P, (lc + 1) * D.chunk_px);
  for (int p = lc * D.chunk_px + threadIdx.x; p < pend; p += kThreads) {
    const float d = expf(D.logd[poff + p]);
    const int v = p / W, u = p - v * W;
    const float c0 = d * (float(u) - iT[14]) * iT[12], c1 = d * (float(v) - iT[15]) * iT[13];
    float* o = out + (poff + p) * 3;
    o[0] = iT[0] * c0 + iT[1] * c1 + iT[2] * d + iT[9];
    o[1] = iT[3] * c0 + iT[4] * c1 + iT[5] * d + iT[10];
    o[2] = iT[6] * c0 + iT[7] * c1 + iT[8] * d + iT[11];
  }
}

}  // namespace align
}  // namespace d3r

namespace d3r { namespace align {
int launch_stream(const d3r_align_desc* desc, int it_begin, int it_end, const GradOut* go, cudaStream_t st);
int launch_stream_split(const d3r_align_desc* desc, int it, bool pixel, const GradOut* go, cudaStream_t st);
int stream_set_debug(unsigned long long* p);
} }

using namespace d3r;
using namespace d3r::align;

extern "C" int d3r_align_set_debug(void* dev_buf) {
  unsigned long long* p = reinterpret_cast<unsigned long long*>(dev_buf);
  D3R_CUDA(cudaMemcpyToSymbol(g_align_dbg, &p, sizeof(p)));
  return stream_set_debug(p);
}

extern "C" int d3r_align_chunk_pixels(void) { return kChunk; }
extern "C" int d3r_sizeof_align_desc(void) { return (int)sizeof(d3r_align_desc); }

extern "C" int64_t d3r_align_workspace_floats(int32_t n_imgs, int32_t n_edges) { return workspace_floats(n_imgs, n_edges); }

// optimizer_state: the call reads the Adam moments, the trainable flags and the schedule (everything but a gradient launch)
static int validate(const d3r_align_desc* d, bool optimizer_state = true) {
  D3R_CHECK_ARG(d != nullptr, "d3r_align: null descriptor");
  D3R_CHECK_ARG(d->n_imgs > 0 && d->n_edges > 0 && d->n_entries == 2 * d->n_edges, "d3r_align: bad sizes");
  D3R_CHECK_ARG(d->n_chunks > 0 && d->max_chunks > 0 && d->max_deg > 0, "d3r_align: bad chunking");
  D3R_CHECK_ARG(d->obs && d->logd && d->small && d->workspace && d->loss_out && d->counters, "d3r_align: null buffer");
  D3R_CHECK_ARG(!optimizer_state || (d->logd_m && d->logd_v && d->small_m && d->small_v && d->small_trainable && d->sched),
                "d3r_align: null buffer");
  D3R_CHECK_ARG(d->chunk_px > 0 && d->chunk_px <= kChunk, "d3r_align: chunk_px=%d must be in [1, %d]", d->chunk_px, kChunk);
  return D3R_OK;
}

extern "C" int d3r_align_prepare(const d3r_align_desc* desc, void* stream) {
  int rc = validate(desc);
  if (rc) return rc;
  prepare_kernel<<<1, kThreads, 0, (cudaStream_t)stream>>>(*desc);
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}

// go == nullptr: iterations [it_begin, it_end); otherwise one gradient launch
template <bool kL2, int PPT>
static int launch_iters(const d3r_align_desc* desc, int it_begin, int it_end, const GradOut* go, cudaStream_t st) {
  const size_t smem = size_t(kStages) * PPT * kThreads * sizeof(float4) + size_t(kEntTile) * kWarps * kEntVals * sizeof(float);
  if (go) return launch_gradient(align_grad_kernel<kL2, PPT>, desc, desc->n_chunks, kThreads, smem, *go, st);
  return launch_iterations(align_iter_kernel<kL2, PPT>, desc, desc->n_chunks, kThreads, smem, it_begin, it_end, st);
}

template <bool kL2>
static int launch_ppt(const d3r_align_desc* desc, int it_begin, int it_end, const GradOut* go, cudaStream_t st) {
  const int ppt = (desc->chunk_px + kThreads - 1) / kThreads;   // pixel slots per thread this problem needs
  if (ppt <= 4) return launch_iters<kL2, 4>(desc, it_begin, it_end, go, st);
  if (ppt == 5) return launch_iters<kL2, 5>(desc, it_begin, it_end, go, st);
  if (ppt == 6) return launch_iters<kL2, 6>(desc, it_begin, it_end, go, st);
  if (ppt == 7) return launch_iters<kL2, 7>(desc, it_begin, it_end, go, st);
  return launch_iters<kL2, 8>(desc, it_begin, it_end, go, st);
}

extern "C" int d3r_align_run(const d3r_align_desc* desc, int32_t it_begin, int32_t it_end, void* stream) {
  int rc = validate(desc);
  if (rc) return rc;
  D3R_CHECK_ARG(it_begin >= 0 && it_end >= it_begin, "d3r_align_run: bad iteration range");
  if (it_begin == 0) {   // the overflow flag reports on the run that starts here
    const Workspace ws0 = carve(desc->workspace, desc->n_imgs, desc->n_edges);
    D3R_CUDA(cudaMemsetAsync(ws0.flags, 0, sizeof(int), (cudaStream_t)stream));
  }
  prof::Scope scope(desc->stream_kernel ? "align_stream" : "align_iter", (cudaStream_t)stream, 0.0, 0.0, it_end - it_begin);
  if (desc->stream_kernel) return launch_stream(desc, it_begin, it_end, nullptr, (cudaStream_t)stream);
  return desc->dist_l2 ? launch_ppt<true>(desc, it_begin, it_end, nullptr, (cudaStream_t)stream)
                       : launch_ppt<false>(desc, it_begin, it_end, nullptr, (cudaStream_t)stream);
}

extern "C" int d3r_align_pixel_pass(const d3r_align_desc* desc, int32_t it, void* stream) {
  int rc = validate(desc);
  if (rc) return rc;
  D3R_CHECK_ARG(it >= 0, "d3r_align_pixel_pass: bad iteration %d", it);
  prof::Scope scope("align_pixel", (cudaStream_t)stream, 0.0, 0.0, 1);
  return launch_stream_split(desc, it, true, nullptr, (cudaStream_t)stream);
}

extern "C" int d3r_align_grad_pixel_pass(const d3r_align_desc* desc, float* logd_grad, void* stream) {
  int rc = validate(desc, false);
  if (rc) return rc;
  D3R_CHECK_ARG(logd_grad, "d3r_align_grad_pixel_pass: null gradient buffer");
  prof::Scope scope("align_grad_pixel", (cudaStream_t)stream, 0.0, 0.0, 1);
  const GradOut go{logd_grad, nullptr, nullptr};
  return launch_stream_split(desc, 0, true, &go, (cudaStream_t)stream);
}

extern "C" int d3r_align_small_step(const d3r_align_desc* desc, int32_t it, void* stream) {
  int rc = validate(desc);
  if (rc) return rc;
  D3R_CHECK_ARG(it >= 0, "d3r_align_small_step: bad iteration %d", it);
  if (it == 0) {   // the overflow flag reports on the run that starts here (only the small step writes it in a split iteration)
    const Workspace ws0 = carve(desc->workspace, desc->n_imgs, desc->n_edges);
    D3R_CUDA(cudaMemsetAsync(ws0.flags, 0, sizeof(int), (cudaStream_t)stream));
  }
  prof::Scope scope("align_small", (cudaStream_t)stream, 0.0, 0.0, 1);
  return launch_stream_split(desc, it, false, nullptr, (cudaStream_t)stream);
}

extern "C" int d3r_align_grad_small_step(const d3r_align_desc* desc, float* small_grad, float* entry_loss, void* stream) {
  int rc = validate(desc, false);
  if (rc) return rc;
  D3R_CHECK_ARG(small_grad, "d3r_align_grad_small_step: null gradient buffer");
  const Workspace ws0 = carve(desc->workspace, desc->n_imgs, desc->n_edges);
  D3R_CUDA(cudaMemsetAsync(ws0.flags, 0, sizeof(int), (cudaStream_t)stream));   // the overflow flag reports on this evaluation
  prof::Scope scope("align_grad_small", (cudaStream_t)stream, 0.0, 0.0, 1);
  const GradOut go{nullptr, small_grad, entry_loss};
  return launch_stream_split(desc, 0, false, &go, (cudaStream_t)stream);
}

extern "C" int d3r_align_reduce_block(int32_t n_imgs, int32_t n_edges, int64_t* offset_floats, int64_t* n_words) {
  D3R_CHECK_ARG(n_imgs > 0 && n_edges > 0 && offset_floats && n_words, "d3r_align_reduce_block: bad arguments");
  reduce_block(n_imgs, n_edges, offset_floats, n_words);
  return D3R_OK;
}

extern "C" int d3r_align_loss_grad(const d3r_align_desc* desc, float* logd_grad, float* small_grad, float* entry_loss, void* stream) {
  int rc = validate(desc, false);
  if (rc) return rc;
  D3R_CHECK_ARG(logd_grad && small_grad, "d3r_align_loss_grad: null gradient buffer");
  const Workspace ws0 = carve(desc->workspace, desc->n_imgs, desc->n_edges);
  D3R_CUDA(cudaMemsetAsync(ws0.flags, 0, sizeof(int), (cudaStream_t)stream));   // the overflow flag reports on this launch
  prof::Scope scope("align_grad", (cudaStream_t)stream, 0.0, 0.0, 1);
  const GradOut go{logd_grad, small_grad, entry_loss};
  if (desc->stream_kernel) return launch_stream(desc, 0, 1, &go, (cudaStream_t)stream);
  return desc->dist_l2 ? launch_ppt<true>(desc, 0, 1, &go, (cudaStream_t)stream) : launch_ppt<false>(desc, 0, 1, &go, (cudaStream_t)stream);
}

/* 1 if a fixed-point accumulator overflowed (|partial sum| >= 2^18) since the flag was last cleared. */
extern "C" int d3r_align_overflow_flag(const d3r_align_desc* desc, int32_t* host_out, void* stream) {
  int rc = validate(desc);
  if (rc) return rc;
  const Workspace ws = carve(desc->workspace, desc->n_imgs, desc->n_edges);
  D3R_CUDA(cudaMemcpyAsync(host_out, ws.flags, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  D3R_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return D3R_OK;
}

extern "C" int d3r_align_pts3d(const d3r_align_desc* desc, float* out_dev, void* stream) {
  int rc = validate(desc);
  if (rc) return rc;
  D3R_CHECK_ARG(out_dev != nullptr, "d3r_align_pts3d: null output");
  pts3d_kernel<<<desc->n_chunks, kThreads, 0, (cudaStream_t)stream>>>(*desc, out_dev);
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}
