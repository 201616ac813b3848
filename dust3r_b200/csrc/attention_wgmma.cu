// wgmma fused attention for head dim 64 (sm_90a): the kernel, its host entry and the C ABI.
//
//   O = softmax(Q K^T * scale) V      per (image b, head h), bf16 in/out, fp32 softmax + accumulation
//   O[b, i, h*64 + d] = softmax_j(scale * q[b,i,h,:] . k[b,j,h,:]) v[b,j,h,d]   replaces the materialised (B,H,N,N) fp32
//   attention matrix of croco/models/blocks.py:105-109 / :161-165.
//
// Flash-attention dataflow on Hopper: a 128-query tile per CTA iteration, 128-key blocks, S and O in registers.
// CTAs are PERSISTENT (1 per SM, 384 threads): each loops over (query tile, head, image) work items, so barrier set-up
// is paid once per CTA and the next tile's Q and K/V loads are already in flight while the current tile finishes.
//
//   warpgroup 0      TMA producer : per tile Q, then K_j / V_j (128 keys x 64) into 2-deep rings
//   warpgroups 1, 2  consumers    : 64 query rows each.  S = Q K_j^T (wgmma m64n128k16 x4, both operands from shared
//                                   memory), online softmax on the S registers (a row lives in the four threads of a
//                                   quad), then O += P V_j (wgmma m64n64k16 x8, B = V_j MN-major).
//
// Two variants of the P V product, which produce the same bits:
//   P_SMEM = false (default)  P stays in registers: the S accumulator fragment, packed to bf16, is exactly the A
//                             fragment of the next wgmma
//   P_SMEM = true             P goes through 128B-swizzled shared memory (both wgmma operands from shared memory);
//                             kept as the A/B reference of the register path, selected by d3r_set_attention_impl(2)
#include "d3r_common.cuh"
#include "sm90_ptx.cuh"
#include "elementwise.h"
#include "prof.h"
#include "pdl.cuh"

namespace d3r {
namespace attn {

namespace wg {

constexpr int BQ = 128, BK = 128, D = 64;
constexpr int kThreads = 384;
constexpr int kTileBytes = 128 * 64 * 2;  // 16 KB: 128 rows x 128 B (Q tile, one K / V block)
constexpr int kPBytes = 2 * 64 * 128 * 2;  // per consumer warpgroup: 64 rows x 128 keys bf16 = two 64-key swizzle atoms
template <bool P_SMEM>
struct Smem {
  static constexpr int kP = P_SMEM ? 2 * kPBytes : 0;
  static constexpr int kBytes = kTileBytes /*Q*/ + 2 * kTileBytes /*K ring*/ + 2 * kTileBytes /*V ring*/ + kP + 128 /*barriers*/ + 1024;
  static_assert(kBytes <= 227 * 1024, "shared memory of one CTA");
};

template <bool P_SMEM>
__global__ void __launch_bounds__(kThreads, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, __nv_bfloat16* __restrict__ out, long long ldo, int Nq, int Nk,
                 int heads, int total_tiles, float scale_log2) {
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzle atoms need 1024-byte alignment
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_q = smem;
  uint8_t* s_k = s_q + kTileBytes;
  uint8_t* s_v = s_k + 2 * kTileBytes;
  uint8_t* s_p = s_v + 2 * kTileBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_p + Smem<P_SMEM>::kP);
  uint64_t* q_full = bars + 0;
  uint64_t* q_empty = bars + 1;   // every S product of the tile has read Q
  uint64_t* k_full = bars + 2;    // [2]
  uint64_t* k_empty = bars + 4;   // [2]
  uint64_t* v_full = bars + 6;    // [2]
  uint64_t* v_empty = bars + 8;   // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nq_tiles = (Nq + BQ - 1) / BQ;
  const int nblk = (Nk + BK - 1) / BK;
  // work item t -> (query tile, head, image); neighbouring CTAs work on the same (image, head) at the same time,
  // so its K / V are fetched from HBM once and then hit in L2
  auto tile_coords = [&](int t, int& q0, int& h, int& b) {
    q0 = (t % nq_tiles) * BQ;
    h = (t / nq_tiles) % heads;
    b = t / (nq_tiles * heads);
  };

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmap_q);
    ptx::prefetch_tmap(&tmap_k);
    ptx::prefetch_tmap(&tmap_v);
    ptx::mbar_init(ptx::smem_u32(q_full), 1);
    ptx::mbar_init(ptx::smem_u32(q_empty), 8);
    for (int s = 0; s < 2; ++s) {
      ptx::mbar_init(ptx::smem_u32(&k_full[s]), 1);
      ptx::mbar_init(ptx::smem_u32(&k_empty[s]), 8);
      ptx::mbar_init(ptx::smem_u32(&v_full[s]), 1);
      ptx::mbar_init(ptx::smem_u32(&v_empty[s]), 8);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  pdl::sync_with_predecessor();   // set-up done; from here on the kernel reads q/k/v written by its predecessor

  if (warp < 4) {
    // ================= TMA producer =================
    ptx::setmaxnreg_dec<24>();
    if (warp == 0 && ptx::elect_one()) {
      uint32_t g = 0, it = 0;   // global key-block counter / tile counter of this CTA (barrier phases run on across tiles)
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x, ++it) {
        int q0, h, b;
        tile_coords(t, q0, h, b);
        ptx::mbar_wait(ptx::smem_u32(q_empty), (it & 1) ^ 1);
        ptx::mbar_arrive_expect_tx(ptx::smem_u32(q_full), kTileBytes);
        ptx::tma_load_3d(ptx::smem_u32(s_q), &tmap_q, ptx::smem_u32(q_full), h * D, q0, b);
        for (int j = 0; j < nblk; ++j, ++g) {
          const int st = g & 1;
          const uint32_t ph = (g >> 1) & 1;
          ptx::mbar_wait(ptx::smem_u32(&k_empty[st]), ph ^ 1);
          ptx::mbar_arrive_expect_tx(ptx::smem_u32(&k_full[st]), kTileBytes);
          ptx::tma_load_3d(ptx::smem_u32(s_k + st * kTileBytes), &tmap_k, ptx::smem_u32(&k_full[st]), h * D, j * BK, b);
          ptx::mbar_wait(ptx::smem_u32(&v_empty[st]), ph ^ 1);
          ptx::mbar_arrive_expect_tx(ptx::smem_u32(&v_full[st]), kTileBytes);
          ptx::tma_load_3d(ptx::smem_u32(s_v + st * kTileBytes), &tmap_v, ptx::smem_u32(&v_full[st]), h * D, j * BK, b);
        }
      }
    }
  } else {
    // ================= consumers =================
    ptx::setmaxnreg_inc<240>();
    const int cw = (threadIdx.x >> 7) - 1;   // consumer warpgroup: query rows [64 cw, 64 cw + 64) of the tile
    const int wq = warp & 3, q = lane & 3;
    uint8_t* s_pw = s_p + cw * kPBytes;
    // accumulator layouts (wgmma m64nN): this thread holds rows r_h = 16 wq + lane/4 + 8h (h = 0, 1) and, in every n8
    // block n, the columns 8n + 2q + e:  S[4n + 2h + e],  O[4n + 2h + e]
    uint32_t g = 0, it = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x, ++it) {
      int q0, h, b;
      tile_coords(t, q0, h, b);
      float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
      float o[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] = 0.f;
      ptx::mbar_wait(ptx::smem_u32(q_full), it & 1);
      const uint64_t dq = ptx::desc_kmajor_sw128(ptx::smem_u32(s_q + cw * 64 * 128));
      for (int j = 0; j < nblk; ++j, ++g) {
        const int st = g & 1;
        const uint32_t ph = (g >> 1) & 1;
        // ---- S = Q K_j^T ----
        float s[64];
        ptx::mbar_wait(ptx::smem_u32(&k_full[st]), ph);
        const uint64_t dk = ptx::desc_kmajor_sw128(ptx::smem_u32(s_k + st * kTileBytes));
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < D / 16; ++k) ptx::wgmma_m64n128k16_ss(s, dq + uint64_t(2 * k), dk + uint64_t(2 * k), k ? 1u : 0u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::reg_fence(s);
        if (lane == 0) {
          ptx::mbar_arrive(ptx::smem_u32(&k_empty[st]));
          if (j == nblk - 1) ptx::mbar_arrive(ptx::smem_u32(q_empty));
        }
        // ---- online softmax ----
        const int nvalid = Nk - j * BK;   // keys past Nk (zero-filled by TMA) get p = 0
        if (nvalid < BK) {
#pragma unroll
          for (int n = 0; n < 16; ++n)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (8 * n + 2 * q + e >= nvalid) { s[4 * n + e] = -INFINITY; s[4 * n + 2 + e] = -INFINITY; }
        }
        float ms[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float mx = -INFINITY;
#pragma unroll
          for (int n = 0; n < 16; ++n) mx = fmaxf(mx, fmaxf(s[4 * n + 2 * hh], s[4 * n + 2 * hh + 1]));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          const float m_new = fmaxf(m_run[hh], mx);   // finite: every block has at least one valid key
          const float corr = ptx::ex2_approx((m_run[hh] - m_new) * scale_log2);
          m_run[hh] = m_new;
          l_run[hh] *= corr;
#pragma unroll
          for (int n = 0; n < 8; ++n) { o[4 * n + 2 * hh] *= corr; o[4 * n + 2 * hh + 1] *= corr; }
          ms[hh] = m_new * scale_log2;
        }
        uint32_t pk[32];   // pk[2n + h]: bf16 pair of row h, keys 8n + 2q, +1;  pk[4kk .. 4kk+3] = A fragment of k-step kk
#pragma unroll
        for (int n = 0; n < 16; ++n)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const float p0 = ptx::ex2_approx(fmaf(s[4 * n + 2 * hh], scale_log2, -ms[hh]));
            const float p1 = ptx::ex2_approx(fmaf(s[4 * n + 2 * hh + 1], scale_log2, -ms[hh]));
            l_run[hh] += p0 + p1;
            pk[2 * n + hh] = pack_bf16x2(p0, p1);
          }
        // ---- O += P V_j ----
        ptx::mbar_wait(ptx::smem_u32(&v_full[st]), ph);
        const uint32_t sv = ptx::smem_u32(s_v + st * kTileBytes);
        if constexpr (P_SMEM) {
          // K-major SW128 atoms of 64 keys: 16-byte chunk index ^ (row & 7)
#pragma unroll
          for (int n = 0; n < 16; ++n)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int r = wq * 16 + (lane >> 2) + 8 * hh;
              *reinterpret_cast<uint32_t*>(s_pw + (n >> 3) * (64 * 128) + r * 128 + (((n & 7) ^ (r & 7)) << 4) + 4 * q) = pk[2 * n + hh];
            }
          ptx::fence_proxy_async();
          asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
          const uint32_t sp = ptx::smem_u32(s_pw);
          ptx::wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < BK / 16; ++kk)
            ptx::wgmma_m64n64k16_ss_tb(o, ptx::desc_kmajor_sw128(sp + (kk >> 2) * (64 * 128)) + uint64_t(2 * (kk & 3)),
                                       ptx::desc_mnmajor_sw128(sv + kk * 16 * 128), 1u);
        } else {
          ptx::wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < BK / 16; ++kk) ptx::wgmma_m64n64k16_rs_tb(o, pk + 4 * kk, ptx::desc_mnmajor_sw128(sv + kk * 16 * 128), 1u);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::reg_fence(o);
        if constexpr (P_SMEM) asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");   // P may be overwritten
        if (lane == 0) ptx::mbar_arrive(ptx::smem_u32(&v_empty[st]));
      }
      // ---- epilogue: O / l -> bf16 -> global ----
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float l = l_run[hh];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = 1.f / l;
        const int qrow = q0 + cw * 64 + wq * 16 + (lane >> 2) + 8 * hh;
        if (qrow < Nq) {
          __nv_bfloat16* orow = out + ((long long)b * Nq + qrow) * ldo + h * D + 2 * q;
#pragma unroll
          for (int n = 0; n < 8; ++n)
            *reinterpret_cast<uint32_t*>(orow + 8 * n) = pack_bf16x2(o[4 * n + 2 * hh] * inv, o[4 * n + 2 * hh + 1] * inv);
        }
      }
    }
  }
}

}  // namespace wg

template <bool P_SMEM>
static int launch_attention(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, void* out, long long ldo, int B, int heads,
                            int Nq, int Nk, float scale, cudaStream_t st) {
  static unsigned long long attr_devices = 0;
  if (first_launch_on_this_device(attr_devices))
    D3R_CUDA(cudaFuncSetAttribute(wg::attention_kernel<P_SMEM>, cudaFuncAttributeMaxDynamicSharedMemorySize, wg::Smem<P_SMEM>::kBytes));
  const int total_tiles = ((Nq + wg::BQ - 1) / wg::BQ) * heads * B;
  const int slots = num_sms();   // one persistent CTA per SM
  // equal number of tiles per CTA where possible: a grid of `slots` CTAs would leave a ragged last round
  const int rounds = (total_tiles + slots - 1) / slots;
  const int grid = (total_tiles + rounds - 1) / rounds;
  prof::Scope scope(P_SMEM ? "attention_wgmma_psmem" : "attention_wgmma", st, 4.0 * double(B) * heads * double(Nq) * double(Nk) * 64.0);
  D3R_CUDA(pdl::launch(wg::attention_kernel<P_SMEM>, dim3(grid), dim3(wg::kThreads), size_t(wg::Smem<P_SMEM>::kBytes), st, mq, mk, mv,
                       (__nv_bfloat16*)out, ldo, Nq, Nk, heads, total_tiles, scale * 1.4426950408889634f));
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}

// tokens of one image: [N][ld] bf16 -> 3-D map {cols, N, B}, box {64, box_rows, 1}: rows past N are zero-filled
static int make_map(CUtensorMap* m, const void* base, long long ld, int cols, int N, int B, int box_rows) {
  const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)N, (cuuint64_t)B};
  const cuuint64_t str[2] = {(cuuint64_t)ld * 2, (cuuint64_t)N * ld * 2};
  const cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
  return encode_tensor_map(m, base, 3, dims, str, box, "attention");
}

// 3 (default): P V with P in registers; 2: the same dataflow with P through shared memory, kept as the A/B reference --
// both produce the same bits.
static int g_impl = 3;

int attention_hd64(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* out,
                   long long ldo, int B, int heads, int Nq, int Nk, float scale, cudaStream_t st) {
  D3R_CHECK_ARG(q && k && v && out && B > 0 && heads > 0 && Nq > 0 && Nk > 0, "attention: bad arguments");
  D3R_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, "attention: row strides must be multiples of 8");
  D3R_CHECK_ARG(((uintptr_t)q & 15) == 0 && ((uintptr_t)k & 15) == 0 && ((uintptr_t)v & 15) == 0 && ((uintptr_t)out & 15) == 0,
                "attention: pointers must be 16-byte aligned");
  CUtensorMap mq, mk, mv;
  int rc;
  if ((rc = make_map(&mq, q, ldq, heads * 64, Nq, B, wg::BQ))) return rc;
  if ((rc = make_map(&mk, k, ldk, heads * 64, Nk, B, wg::BK))) return rc;
  if ((rc = make_map(&mv, v, ldv, heads * 64, Nk, B, wg::BK))) return rc;
  if (g_impl == 2) return launch_attention<true>(mq, mk, mv, out, ldo, B, heads, Nq, Nk, scale, st);
  return launch_attention<false>(mq, mk, mv, out, ldo, B, heads, Nq, Nk, scale, st);
}

}  // namespace attn
}  // namespace d3r

extern "C" void d3r_set_attention_impl(int32_t impl) { d3r::attn::g_impl = (impl == 2) ? 2 : 3; }

extern "C" int d3r_attention_hd64(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out,
                                  int64_t ldo, int32_t B, int32_t heads, int32_t Nq, int32_t Nk, float scale, void* stream) {
  return d3r::attn::attention_hd64(q, ldq, k, ldk, v, ldv, out, ldo, B, heads, Nq, Nk, scale, (cudaStream_t)stream);
}
