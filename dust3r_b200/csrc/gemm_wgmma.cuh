// Persistent warp-specialised bf16 GEMM / implicit-GEMM convolution on wgmma (sm_90a).
//
//   D[M,N] = A[M,K] * B[N,K]^T   (both operands K-major, fp32 accumulation in registers)
//
// Roles (384 threads = three warpgroups, 1 CTA / SM, grid = min(#tiles, #SMs), static round-robin tile schedule with
// the N index fastest so the CTAs of one wave share A rows through L2):
//   warpgroup 0     TMA producer : one elected thread, cp.async.bulk.tensor -> 128B-swizzled smem ring (kStages deep);
//                                  it runs ahead into the next tile while the consumers drain the current one
//   warpgroups 1,2  consumers    : wgmma m64 x BLOCK_N x k16 on rows [64 (wg-1), 64 wg) of the 128-row tile, then the
//                                  fused epilogue from the accumulator registers -> global, either stored straight
//                                  from the registers or (TMA_STORE) staged in shared memory and written by TMA while
//                                  the consumers go on to the next tile
//
// CTA pairs (PAIR = true): a cluster of two CTAs works on two M tiles that share one N tile; each CTA loads half of the
// B tile and multicasts it into both CTAs' shared memory, so B crosses L2 -> SM once per pair.  A ring slot is refilled
// only after the consumers of BOTH CTAs have released it (the empty barriers count the arrivals of both).
//
// A-operand sources: plain row-major [M,K] (2D tensor map), or NHWC activations walked as a 3x3
// convolution (4D tensor map, one box per filter tap; TMA out-of-bounds zero fill = zero padding).
//
// Fused epilogues (runtime flags): +bias, GELU(erf), ReLU, bf16/f32 store, in-place fp32 residual
// accumulate, up to two bf16 addends, dual (raw + ReLU) store, 2D RoPE on q/k columns (replaces
// croco/models/curope), k==stride transposed-conv pixel scatter, and the DPT "head.4 1x1 conv +
// postprocess" tail (dust3r/heads/postprocess.py) evaluated straight from the accumulator.
#pragma once
#include "d3r_common.cuh"
#include "sm90_ptx.cuh"
#include "pdl.cuh"

namespace d3r {
namespace gemm {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;   // 64 bf16 = 128 B = one swizzle atom row
constexpr int WGMMA_K = 16;
constexpr int kNumThreads = 384;
constexpr int kConsumerWarps = 8;

enum : uint32_t {
  F_BIAS = 1u << 0,
  F_GELU = 1u << 1,
  F_RELU = 1u << 2,
  F_OUT_F32 = 1u << 3,        // store fp32 instead of bf16
  F_RESID_INPLACE = 1u << 4,  // out (fp32) += result  (residual stream update)
  F_ADD0 = 1u << 5,           // + bf16 addend 0 (same indexing as out)
  F_ADD1 = 1u << 6,           // + bf16 addend 1
  F_OUT2_RELU = 1u << 7,      // also store relu(result) as bf16 to out2
  F_ROPE = 1u << 8,           // rotate columns < rope_cols (q / k heads of 64)
  F_CONVT = 1u << 9,          // kernel==stride transposed conv scatter
  F_HEAD_FINAL = 1u << 10,    // relu -> 1x1 conv to 4 ch -> pts3d/conf postprocess
  F_OUT2_BF16 = 1u << 11,     // also store the result as bf16 to out2 (used with fp32 primary)
};

struct Params {
  int M, N, K;
  int num_kb;
  int mode;  // 0 plain, 1 conv3x3 (stride 1, pad 1)
  uint32_t flags;
  void* out;
  void* out2;
  const void* add0;
  const void* add1;
  const float* bias;
  long long ldo;
  // RoPE
  const float* rope_cos;  // [max_pos][16]
  const float* rope_sin;
  int rope_cols, tokens_per_img, grid_w;
  // conv geometry
  int cB, cH, cW, cin_blocks, tile_w, tile_h, tiles_x, tiles_y;
  // transposed conv (k == stride): A rows are input pixels (b, iy, ix)
  int tk, th_in, tw_in, tCout;
  // head tail
  const float* w4;  // [4][128]
  const float* b4;  // [4]
  float* pts3d;     // (B,H,W,3)
  float* conf;      // (B,H,W)
  int depth_mode;   // 0 linear, 1 square, 2 exp
  int conf_mode;    // 0 none, 1 exp, 2 sigmoid
  float conf_min, conf_max;
};

// Epilogue specialisations (compile-time): the runtime flag word is masked with the set a specialisation supports,
// so the other epilogue branches are dead code and do not cost registers or instruction cache.
//   EPI_GENERIC  every flag (conv, transposed conv, DPT fusions, head tail, ...)
//   EPI_RESID    out(f32) += acc + bias (the residual stream update)
//   EPI_ACT      bias / GELU / ReLU -> bf16
//   EPI_ROPE     bias + 2D RoPE -> bf16 (q,k,v projections)
//   EPI_CONV     the DPT 3x3 convolutions: bias, up to two bf16 addends, ReLU, raw + ReLU copy (conv_kernel only; the
//                launch is reported as the generic epilogue, whose conv launches it replaces)
enum : int { EPI_GENERIC = 0, EPI_RESID = 1, EPI_ACT = 2, EPI_ROPE = 3, EPI_CONV = 4 };
template <int EPI> struct EpiMask { static constexpr uint32_t value = 0xFFFFFFFFu; };
template <> struct EpiMask<EPI_RESID> { static constexpr uint32_t value = F_BIAS | F_RESID_INPLACE; };
template <> struct EpiMask<EPI_ACT> { static constexpr uint32_t value = F_BIAS | F_GELU | F_RELU; };
template <> struct EpiMask<EPI_ROPE> { static constexpr uint32_t value = F_BIAS | F_ROPE; };
template <> struct EpiMask<EPI_CONV> { static constexpr uint32_t value = F_BIAS | F_RELU | F_ADD0 | F_ADD1 | F_OUT2_RELU; };

// The conv epilogue's other NHWC tensors (B,H,W,Cout) bf16, as 4D tensor maps with boxes of 64 channels x one
// warpgroup's 64 pixels: out2 (F_OUT2_RELU), add0 (F_ADD0), add1 (F_ADD1).  Maps a launch does not use are not read.
struct ConvMaps {
  CUtensorMap out2, add0, add1;
};

__host__ __device__ inline int pick_epi(int mode, uint32_t flags) {
  if (mode != 0) return EPI_GENERIC;
  if ((flags & ~F_BIAS) == F_RESID_INPLACE) return EPI_RESID;
  if ((flags & ~EpiMask<EPI_ACT>::value) == 0) return EPI_ACT;
  if ((flags & ~EpiMask<EPI_ROPE>::value) == 0) return EPI_ROPE;
  return EPI_GENERIC;
}

// Shared memory: the ring, then (TMA_STORE) the epilogue's staging buffers, two per consumer warpgroup, each 64 rows of
// 128 B; then the barriers and (register-store kernels) the head tail's weights, which only EPI_GENERIC reads.
template <int BLOCK_N, bool TMA_STORE = false>
struct Cfg {
  static constexpr int kStageA = BLOCK_M * BLOCK_K * 2;
  static constexpr int kStageB = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStages = (BLOCK_N == 256) ? 4 : (BLOCK_N == 128) ? 6 : 8;
  static constexpr int kRing = kStages * (kStageA + kStageB);
  static constexpr int kOutBuf = 64 * 128;
  static constexpr int kStaging = TMA_STORE ? 2 * 2 * kOutBuf : 0;
  static constexpr int kSmemBytes = kRing + kStaging + 1024 /*align*/ + 256 /*barriers*/ + (TMA_STORE ? 0 : (4 * 128 + 16) * 4) /*head*/;
  static_assert(kSmemBytes <= 227 * 1024, "shared memory of one CTA");
};

// exact-erf GELU (nn.GELU default).  erf by Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, far below the
// bf16 rounding of the stored activation).  Written for the epilogue's instruction budget (14 per element, two
// of them MUFU): with u = |x| sqrt(log2(e)/2),  exp(-x^2/2) = 2^(-u u);  h = x/2 poly(t) t 2^(-u u) (the 1/2 is
// folded into the coefficients) is x/2 (1 - erf(|x|/sqrt2)), and  gelu(x) = max(x, 0) - |h|  on both sides of 0.
__device__ __forceinline__ float gelu_erf(float x) {
  constexpr float kU = 0.84932180028801904f;            // sqrt(log2(e) / 2)
  constexpr float kP = 0.3275911f * 0.70710678118654752f / kU;
  const float u = fabsf(x) * kU;
  const float t = ptx::rcp_approx(fmaf(kP, u, 1.f));
  float poly = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
  poly = fmaf(poly, t, 0.5f * 1.421413741f);
  poly = fmaf(poly, t, 0.5f * -0.284496736f);
  poly = fmaf(poly, t, 0.5f * 0.254829592f);
  const float e = ptx::ex2_approx(-u * u);
  const float h = x * (poly * t * e);
  return fmaxf(x, 0.f) - fabsf(h);
}

// TMA_STORE (specialised projection epilogues at BLOCK_N = 256, the conv epilogue at BLOCK_N = 256 / 128): the epilogue
// stages the tile in shared memory 64 rows at a time and one thread per warpgroup writes it with a TMA store (bf16) or TMA
// reduce-add (EPI_RESID) through tmap_o, which the register-store kernels do not read.  cm: EPI_CONV only.
// The body of gemm_kernel and conv_kernel (below): producer, main loop and every epilogue.
template <int BLOCK_N, int EPI, bool PAIR, bool TMA_STORE>
__device__ __forceinline__ void gemm_body(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, const CUtensorMap& tmap_o,
                                          const ConvMaps* cm, const Params& p) {
  static_assert(EPI == EPI_CONV ? (TMA_STORE && (BLOCK_N == 256 || BLOCK_N == 128))
                                : (!TMA_STORE || (BLOCK_N == 256 && EPI != EPI_GENERIC)),
                "TMA-store epilogue: specialised projection epilogues on 128x256 tiles, the conv epilogue on 128x256 / 128x128");
  using C = Cfg<BLOCK_N, TMA_STORE>;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the 128B swizzle atoms (the same offset in both CTAs of a pair: multicast writes by offset)
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + C::kStages * C::kStageA;
  uint8_t* smem_o = smem + C::kRing;              // [2 warpgroups][2 buffers][64 rows][128 B] (TMA_STORE)
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::kRing + C::kStaging);
  uint64_t* full_bar = bars;                      // [kStages]
  uint64_t* empty_bar = bars + C::kStages;        // [kStages]
  uint64_t* add_bar = bars + 2 * C::kStages;      // [2 warpgroups] (EPI_CONV: addend chunks landed)
  float* s_w4 = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);  // [4][128] + [4]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = PAIR ? ptx::cluster_ctarank() : 0u;
  const int n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int m_tiles = (p.mode == 1) ? p.cB * p.tiles_y * p.tiles_x : (p.M + BLOCK_M - 1) / BLOCK_M;
  // both CTAs of a pair walk the same schedule of (M-tile pair, N tile) work items
  const int m_groups = PAIR ? (m_tiles + 1) / 2 : m_tiles;
  const int total_items = m_groups * n_tiles;
  const int first_item = PAIR ? blockIdx.x / 2 : blockIdx.x;
  const int item_stride = PAIR ? gridDim.x / 2 : gridDim.x;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmap_a);
    ptx::prefetch_tmap(&tmap_b);
    if constexpr (TMA_STORE) ptx::prefetch_tmap(&tmap_o);
    for (int s = 0; s < C::kStages; ++s) {
      ptx::mbar_init(ptx::smem_u32(&full_bar[s]), 1);
      ptx::mbar_init(ptx::smem_u32(&empty_bar[s]), (PAIR ? 2 : 1) * kConsumerWarps);
    }
    if constexpr (EPI == EPI_CONV) {
      ptx::prefetch_tmap(&cm->out2);
      ptx::prefetch_tmap(&cm->add0);
      ptx::prefetch_tmap(&cm->add1);
      ptx::mbar_init(ptx::smem_u32(&add_bar[0]), 1);
      ptx::mbar_init(ptx::smem_u32(&add_bar[1]), 1);
    }
    ptx::fence_barrier_init();
  }
  if (!TMA_STORE && (p.flags & F_HEAD_FINAL) && threadIdx.x >= 128) {
    for (int i = threadIdx.x - 128; i < 4 * 128 + 4; i += 256) s_w4[i] = (i < 512) ? p.w4[i] : p.b4[i - 512];
  }
  __syncthreads();
  if constexpr (PAIR) ptx::cluster_sync();   // the partner's barriers exist before anything is multicast into it
  pdl::sync_with_predecessor();   // set-up done (weights-only reads so far); A / residual / addends come from other kernels

  if (warp < 4) {
    // ================= TMA producer =================
    ptx::setmaxnreg_dec<40>();
    if (warp == 0 && ptx::elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int item = first_item; item < total_items; item += item_stride) {
        const int tn = item % n_tiles, tm = (item / n_tiles) * (PAIR ? 2 : 1) + int(rank);
        int cb = 0, cy0 = 0, cx0 = 0;
        if (p.mode == 1) {
          cb = tm / (p.tiles_y * p.tiles_x);
          const int r = tm - cb * (p.tiles_y * p.tiles_x);
          cy0 = (r / p.tiles_x) * p.tile_h;
          cx0 = (r % p.tiles_x) * p.tile_w;
        }
        for (int kb = 0; kb < p.num_kb; ++kb) {
          ptx::mbar_wait(ptx::smem_u32(&empty_bar[stage]), phase ^ 1);
          const uint32_t fb = ptx::smem_u32(&full_bar[stage]);
          ptx::mbar_arrive_expect_tx(fb, C::kStageA + C::kStageB);
          const uint32_t sa = ptx::smem_u32(smem_a + stage * C::kStageA);
          const uint32_t sb = ptx::smem_u32(smem_b + stage * C::kStageB);
          int ka, kt = 0;
          if (p.mode == 1) {
            const int tap = kb / p.cin_blocks, cblk = kb - tap * p.cin_blocks;
            const int dy = tap / 3, dx = tap - dy * 3;
            ptx::tma_load_4d(sa, &tmap_a, fb, cblk * BLOCK_K, cx0 + dx - 1, cy0 + dy - 1, cb);
            ka = cblk * BLOCK_K;
            kt = tap;
          } else {
            ptx::tma_load_2d(sa, &tmap_a, fb, kb * BLOCK_K, tm * BLOCK_M);
            ka = kb * BLOCK_K;
          }
          if constexpr (PAIR) {
            constexpr int kHalf = BLOCK_N / 2;
            ptx::tma_load_3d_mc(sb + rank * (kHalf * BLOCK_K * 2), &tmap_b, fb, ka, kt, tn * BLOCK_N + int(rank) * kHalf, 0x3);
          } else {
            ptx::tma_load_3d(sb, &tmap_b, fb, ka, kt, tn * BLOCK_N);
          }
          if (++stage == C::kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ================= consumers: wgmma + epilogue =================
    ptx::setmaxnreg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;   // 0: rows [0,64) of the tile, 1: rows [64,128)
    const int wq = warp & 3;
    const int q = lane & 3;
    const uint32_t flags = p.flags & EpiMask<EPI>::value;
    constexpr int kNB = BLOCK_N / 8;         // n8 blocks of the accumulator
    float acc[BLOCK_N / 2];
    int stage = 0;
    uint32_t phase = 0;
    uint32_t out_chunk = 0;                  // TMA_STORE: chunks this warpgroup has staged so far (buffer = out_chunk & 1)
    auto release = [&](int s) {
      if (lane == 0) {
        if constexpr (PAIR) {
          ptx::mbar_arrive_cluster(ptx::smem_u32(&empty_bar[s]), 0);
          ptx::mbar_arrive_cluster(ptx::smem_u32(&empty_bar[s]), 1);
        } else {
          ptx::mbar_arrive(ptx::smem_u32(&empty_bar[s]));
        }
      }
    };
    // EPI_CONV: this warpgroup's 64 pixels of conv tile tm are one (64 ch, bw, bh, 1) box of the NHWC output maps at
    // (x, y, b) = conv_box(tm) (bw = min(tile_w, 64), bh = 64 / bw): row r of the box is row 64 wg + r of the tile.  Pixels
    // past W / H, and the missing M tile of an odd count in the CTA pair, lie outside the maps and are not written.
    const bool conv_issuer = EPI == EPI_CONV && (threadIdx.x & 127) == 0;
    const bool conv_two = EPI == EPI_CONV && (flags & (F_OUT2_RELU | F_ADD1)) != 0;   // two staging buffers per chunk (else one, alternating)
    const bool conv_add = EPI == EPI_CONV && (flags & (F_ADD0 | F_ADD1)) != 0;
    uint32_t add_phase = 0;
    auto conv_box = [&](int tm, int& bx, int& by, int& bb) {
      bb = tm / (p.tiles_y * p.tiles_x);
      const int r = tm - bb * (p.tiles_y * p.tiles_x);
      bx = (r % p.tiles_x) * p.tile_w + (64 * wg) % p.tile_w;
      by = (r / p.tiles_x) * p.tile_h + (64 * wg) / p.tile_w;
    };
    auto out_buf = [&](int i) { return ptx::smem_u32(smem_o + (wg * 2 + i) * C::kOutBuf); };
    // (conv_issuer) TMA-load the addends of channels [ch, ch + 64) of tile tm into the buffer(s) that chunk is staged in, once
    // the stores that last read them are done; completion on add_bar[wg]
    auto issue_addends = [&](int tm, int ch) {
      int bx, by, bb;
      conv_box(tm, bx, by, bb);
      const uint32_t b0 = conv_two ? out_buf(0) : out_buf(out_chunk & 1);
      if (conv_two) ptx::bulk_wait_group_read<0>();
      else ptx::bulk_wait_group_read<1>();
      const uint32_t bar = ptx::smem_u32(&add_bar[wg]);
      ptx::mbar_arrive_expect_tx(bar, uint32_t(C::kOutBuf) * (((flags & F_ADD0) ? 1u : 0u) + ((flags & F_ADD1) ? 1u : 0u)));
      if (flags & F_ADD0) ptx::tma_load_4d(b0, &cm->add0, bar, ch, bx, by, bb);
      if (flags & F_ADD1) ptx::tma_load_4d(out_buf(1), &cm->add1, bar, ch, bx, by, bb);
    };
    for (int item = first_item; item < total_items; item += item_stride) {
      const int tn = item % n_tiles, tm = (item / n_tiles) * (PAIR ? 2 : 1) + int(rank);
      if constexpr (EPI == EPI_CONV) {
        if (conv_add && conv_issuer) issue_addends(tm, tn * BLOCK_N);   // lands while the main loop runs
      }
      // ---- main loop: one wgmma group per k-block; a slot is released once the group after it has been issued ----
      int prev = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        ptx::mbar_wait(ptx::smem_u32(&full_bar[stage]), phase);
        const uint64_t da = ptx::desc_kmajor_sw128(ptx::smem_u32(smem_a + stage * C::kStageA + wg * 64 * 128));
        const uint64_t db = ptx::desc_kmajor_sw128(ptx::smem_u32(smem_b + stage * C::kStageB));
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k) {
          // advance 32 B (= 16 bf16 of K) inside the 128 B swizzle row: +2 in 16-byte units
          if constexpr (BLOCK_N == 256) ptx::wgmma_m64n256k16_ss(acc, da + uint64_t(2 * k), db + uint64_t(2 * k), (kb | k) != 0 ? 1u : 0u);
          else if constexpr (BLOCK_N == 128) ptx::wgmma_m64n128k16_ss(acc, da + uint64_t(2 * k), db + uint64_t(2 * k), (kb | k) != 0 ? 1u : 0u);
          else ptx::wgmma_m64n64k16_ss(acc, da + uint64_t(2 * k), db + uint64_t(2 * k), (kb | k) != 0 ? 1u : 0u);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == C::kStages) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      ptx::reg_fence(acc);
      release(prev);

      // ---- epilogue.  Accumulator layout of wgmma m64nN: this thread holds rows (wq*16 + lane/4) and (+8) of its
      // warpgroup's 64, and in every n8 block j the two columns 8j + 2q, 8j + 2q + 1:
      //   acc[4j + 2h + e] = D[row_h][8j + 2q + e]
      bool valid[2];
      long long row_off[2];
      int tok[2] = {0, 0};
      long long pix[2] = {0, 0};
      int ct_b[2] = {0, 0}, ct_iy[2] = {0, 0}, ct_ix[2] = {0, 0};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row_in_tile = wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
        if (p.mode == 1) {
          const int cb = tm / (p.tiles_y * p.tiles_x);
          const int r = tm - cb * (p.tiles_y * p.tiles_x);
          const int y = (r / p.tiles_x) * p.tile_h + row_in_tile / p.tile_w;
          const int x = (r % p.tiles_x) * p.tile_w + row_in_tile % p.tile_w;
          valid[h] = (tm < m_tiles) && (y < p.cH) && (x < p.cW);
          pix[h] = (long long)(cb * p.cH + y) * p.cW + x;
          row_off[h] = pix[h] * p.ldo;
        } else {
          const int row = tm * BLOCK_M + row_in_tile;
          valid[h] = row < p.M;
          row_off[h] = (long long)row * p.ldo;
          if (flags & F_ROPE) tok[h] = row % p.tokens_per_img;
          if (flags & F_CONVT) {
            ct_b[h] = row / (p.th_in * p.tw_in);
            const int r = row - ct_b[h] * (p.th_in * p.tw_in);
            ct_iy[h] = r / p.tw_in;
            ct_ix[h] = r - ct_iy[h] * p.tw_in;
          }
        }
      }
      // (1) bias, GELU
      if (flags & (F_BIAS | F_GELU)) {
#pragma unroll
        for (int j = 0; j < kNB; ++j) {
          const int c = tn * BLOCK_N + 8 * j + 2 * q;
          float2 b = make_float2(0.f, 0.f);
          if ((flags & F_BIAS) && c < p.N) {
            if (flags & F_CONVT) b = make_float2(__ldg(p.bias + c % p.tCout), __ldg(p.bias + (c + 1) % p.tCout));
            else b = __ldg(reinterpret_cast<const float2*>(p.bias + c));
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float& v0 = acc[4 * j + 2 * h];
            float& v1 = acc[4 * j + 2 * h + 1];
            v0 += b.x;
            v1 += b.y;
            if (flags & F_GELU) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
          }
        }
      }
      // (2) RoPE: every 32-column chunk is one half (y or x) of a 64-wide head: pairs (k, k+16) of the chunk, angle =
      //     pos * base^(-k/16); column k + 16 sits two n8 blocks further in the same thread
      if (flags & F_ROPE) {
#pragma unroll
        for (int cb = 0; cb < BLOCK_N / 32; ++cb) {
          const int col0 = tn * BLOCK_N + cb * 32;
          if (col0 >= p.rope_cols) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int pos = ((col0 & 63) < 32) ? (tok[h] / p.grid_w) : (tok[h] % p.grid_w);
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
              const int k = 8 * jj + 2 * q;
              const float2 cs = __ldg(reinterpret_cast<const float2*>(p.rope_cos + pos * 16 + k));
              const float2 sn = __ldg(reinterpret_cast<const float2*>(p.rope_sin + pos * 16 + k));
              const float cc[2] = {cs.x, cs.y}, ss[2] = {sn.x, sn.y};
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                float& u = acc[(4 * cb + jj) * 4 + 2 * h + e];
                float& w = acc[(4 * cb + jj + 2) * 4 + 2 * h + e];
                const float u0 = u, w0 = w;
                u = u0 * cc[e] - w0 * ss[e];
                w = w0 * cc[e] + u0 * ss[e];
              }
            }
          }
        }
      }
      if constexpr (EPI == EPI_CONV) {
        // (3) conv: the warpgroup's 64 pixels x BLOCK_N channels leave in chunks of 64 channels, one tensor-map box each,
        //     staged in the 128B-swizzled layout of the projections' chunks below.  The addends arrive by TMA in the
        //     buffer the chunk is staged in (add1 in the second one) and are replaced in place by the result; out2 =
        //     relu(result) leaves through the second buffer.  With one buffer per chunk (no add1 / out2) the two buffers
        //     alternate between chunks.  Same arithmetic order as the register path: acc + bias, + add0, + add1, ReLU.
        int bx, by, bb;
        conv_box(tm, bx, by, bb);
        const uint32_t sw = lane >> 2;           // (row & 7) of both rows this thread holds
#pragma unroll
        for (int c = 0; c < BLOCK_N / 64; ++c) {
          const uint32_t b0 = conv_two ? out_buf(0) : out_buf(out_chunk & 1), b1 = out_buf(1);
          if (conv_add) {
            ptx::mbar_wait(ptx::smem_u32(&add_bar[wg]), add_phase);
            add_phase ^= 1;
          } else if (conv_two) {
            if (conv_issuer) ptx::bulk_wait_group_read<0>();   // both buffers free again
            ptx::named_bar_sync(1 + wg, 128);
          }
#pragma unroll
          for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t off = (wq * 16 + (lane >> 2) + 8 * h) * 128 + ((j ^ sw) << 4) + q * 4;
              float v0 = acc[4 * (c * 8 + j) + 2 * h], v1 = acc[4 * (c * 8 + j) + 2 * h + 1];
              if (flags & F_ADD0) {
                const float2 a = bf16x2_to_float2(ptx::ld_shared_b32(b0 + off));
                v0 += a.x; v1 += a.y;
              }
              if (flags & F_ADD1) {
                const float2 a = bf16x2_to_float2(ptx::ld_shared_b32(b1 + off));
                v0 += a.x; v1 += a.y;
              }
              if (flags & F_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
              ptx::st_shared_b32(b0 + off, pack_bf16x2(v0, v1));
              if (flags & F_OUT2_RELU) ptx::st_shared_b32(b1 + off, pack_bf16x2(fmaxf(v0, 0.f), fmaxf(v1, 0.f)));
            }
          ptx::fence_proxy_async();
          if (!conv_add && !conv_two && conv_issuer) ptx::bulk_wait_group_read<0>();   // the other buffer free for chunk c + 1
          ptx::named_bar_sync(1 + wg, 128);
          const int ch = tn * BLOCK_N + c * 64;
          if (conv_issuer) {
            ptx::tma_store_4d(&tmap_o, b0, ch, bx, by, bb);
            if (flags & F_OUT2_RELU) ptx::tma_store_4d(&cm->out2, b1, ch, bx, by, bb);
            ptx::bulk_commit_group();
          }
          ++out_chunk;
          if (conv_add && conv_issuer && c + 1 < BLOCK_N / 64) issue_addends(tm, ch + 64);
        }
        continue;
      }
      if constexpr (TMA_STORE) {
        // (3) staged stores: the warpgroup's 64 x 256 result leaves in chunks of 64 rows x 128 B (64 bf16 or 32 fp32
        //     columns), each written into a 128B-swizzled buffer (16-byte unit u of row r at u ^ (r & 7), the layout the
        //     tensor map's swizzle expects) and handed to the TMA unit by thread 0 of the warpgroup.  Two buffers
        //     alternate.  Before the barrier that hands chunk i over, thread 0 waits until chunk i - 1's transfer has read
        //     its buffer, so the barrier also frees that buffer for chunk i + 1.  The transfers of a tile's last chunks
        //     overlap the next tile's main loop; rows past M are clipped by the tensor map.
        constexpr bool kF32 = (EPI == EPI_RESID);
        constexpr int kChunkCols = kF32 ? 32 : 64;
        constexpr int kChunkNB = kChunkCols / 8;
        const bool issuer = (threadIdx.x & 127) == 0;
        const uint32_t sw = lane >> 2;           // (row & 7) of both rows this thread holds
#pragma unroll
        for (int c = 0; c < BLOCK_N / kChunkCols; ++c) {
          const uint32_t buf = ptx::smem_u32(smem_o + (wg * 2 + (out_chunk & 1)) * C::kOutBuf);
#pragma unroll
          for (int j = 0; j < kChunkNB; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t row = wq * 16 + (lane >> 2) + 8 * h;
              float v0 = acc[4 * (c * kChunkNB + j) + 2 * h], v1 = acc[4 * (c * kChunkNB + j) + 2 * h + 1];
              if (flags & F_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
              if constexpr (kF32) {
                // columns 8j + 2q, +1: bytes 32j + 8q of the row
                ptx::st_shared_v2_f32(buf + row * 128 + (((2 * j + (q >> 1)) ^ sw) << 4) + (q & 1) * 8, v0, v1);
              } else {
                ptx::st_shared_b32(buf + row * 128 + ((j ^ sw) << 4) + q * 4, pack_bf16x2(v0, v1));
              }
            }
          ptx::fence_proxy_async();
          if (issuer) ptx::bulk_wait_group_read<0>();
          ptx::named_bar_sync(1 + wg, 128);
          if (issuer) {
            const int c0 = tn * BLOCK_N + c * kChunkCols, r0 = tm * BLOCK_M + wg * 64;
            if constexpr (kF32) ptx::tma_reduce_add_2d(&tmap_o, buf, c0, r0);
            else ptx::tma_store_2d(&tmap_o, buf, c0, r0);
            ptx::bulk_commit_group();
          }
          ++out_chunk;
        }
        continue;
      }
      if (flags & F_HEAD_FINAL) {
        // relu(conv) . w4 over the 128 channels of a row (the whole row is in this tile): this thread's 32 columns,
        // then the four threads of a row quad
        float head_acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
        for (int j = 0; j < kNB; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float r = fmaxf(acc[4 * j + 2 * h + e], 0.f);
              const int c = 8 * j + 2 * q + e;
#pragma unroll
              for (int o = 0; o < 4; ++o) head_acc[h][o] += r * s_w4[o * 128 + c];
            }
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int o = 0; o < 4; ++o) {
            head_acc[h][o] += __shfl_xor_sync(0xffffffffu, head_acc[h][o], 1);
            head_acc[h][o] += __shfl_xor_sync(0xffffffffu, head_acc[h][o], 2);
          }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!valid[h] || q != 0) continue;
          postprocess_pixel(head_acc[h][0] + s_w4[512 + 0], head_acc[h][1] + s_w4[512 + 1], head_acc[h][2] + s_w4[512 + 2],
                            [&] { return head_acc[h][3] + s_w4[512 + 3]; }, p.pts3d, p.conf, pix[h], p.depth_mode, p.conf_mode,
                            p.conf_min, p.conf_max);
        }
        continue;
      }
      // (3) addends, ReLU, stores: two consecutive columns per thread and row
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!valid[h]) continue;
#pragma unroll
        for (int j = 0; j < kNB; ++j) {
          const int col = tn * BLOCK_N + 8 * j + 2 * q;
          if (col >= p.N) continue;
          float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          long long off;
          if (flags & F_CONVT) {
            const int kk = col / p.tCout, co = col - kk * p.tCout;
            const int ky = kk / p.tk, kx = kk - ky * p.tk;
            off = ((long long)(ct_b[h] * p.th_in * p.tk + ct_iy[h] * p.tk + ky) * (p.tw_in * p.tk) + ct_ix[h] * p.tk + kx) * p.tCout + co;
          } else {
            off = row_off[h] + col;
          }
          if (flags & F_ADD0) {
            const float2 a = bf16x2_to_float2(__ldg(reinterpret_cast<const unsigned int*>(reinterpret_cast<const __nv_bfloat16*>(p.add0) + off)));
            v0 += a.x; v1 += a.y;
          }
          if (flags & F_ADD1) {
            const float2 a = bf16x2_to_float2(__ldg(reinterpret_cast<const unsigned int*>(reinterpret_cast<const __nv_bfloat16*>(p.add1) + off)));
            v0 += a.x; v1 += a.y;
          }
          if (flags & F_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          if (flags & (F_OUT_F32 | F_RESID_INPLACE)) {
            float2* o = reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + off);
            if (flags & F_RESID_INPLACE) {
              const float2 r = *o;
              v0 += r.x; v1 += r.y;
            }
            *o = make_float2(v0, v1);
            if (flags & F_OUT2_BF16) *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.out2) + off) = pack_bf16x2(v0, v1);
          } else {
            *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.out) + off) = pack_bf16x2(v0, v1);
            if (flags & F_OUT2_RELU)
              *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.out2) + off) = pack_bf16x2(fmaxf(v0, 0.f), fmaxf(v1, 0.f));
          }
        }
      }
    }
    // the output is complete when the grid is: a dependent launch (PDL) starts on that guarantee
    if constexpr (TMA_STORE) {
      if ((threadIdx.x & 127) == 0) ptx::bulk_wait_group<0>();
    }
  }
  if constexpr (PAIR) ptx::cluster_sync();   // no CTA leaves while its partner may still arrive on its barriers
}

template <int BLOCK_N, int EPI, bool PAIR, bool TMA_STORE>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_o, const Params p) {
  gemm_body<BLOCK_N, EPI, PAIR, TMA_STORE>(tmap_a, tmap_b, tmap_o, nullptr, p);
}

// The DPT 3x3 convolutions (mode 1) with the staged conv epilogue (EPI_CONV): BLOCK_N = Cout = 256 or 128, output
// through the 4D map tmap_o, out2 / addends through cm.
template <int BLOCK_N, bool PAIR>
__global__ void __launch_bounds__(kNumThreads, 1)
conv_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_o, const __grid_constant__ ConvMaps cm, const Params p) {
  gemm_body<BLOCK_N, EPI_CONV, PAIR, true>(tmap_a, tmap_b, tmap_o, &cm, p);
}

}  // namespace gemm
}  // namespace d3r
