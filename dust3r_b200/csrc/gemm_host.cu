// Host side of the wgmma GEMM / conv kernels: tensor-map construction, tile-shape selection, launch.
#include "gemm_wgmma.cuh"
#include "gemm_host.h"
#include "prof.h"

namespace d3r {
namespace gemm {

// conv_m_tiles > 0: a 3x3 conv with the staged epilogue (Cout 256 or 128) over that many 128-pixel tiles.  A 128x256 tile
// holds all 256 output channels, so each A tile is read once instead of once per 128-channel half, at 7.6 instead of
// 11.4 KB of operands per MFLOP.  It is used when there are at least 4 waves of CTA-pair work items at that width
// (levels 0 and 1 of the DPT head at B = 32: 1536 and 384 items for 66 pairs).  With fewer, the partly filled last wave
// of double-size items costs more than the operand traffic saves (level 2: 96 items, i.e. 2 rounds of 256-wide items
// against 3 of 128-wide ones, which take half as long; level 3: 32 items, half the SMs idle), and 128x128 tiles are used.
static int pick_block_n(int N, int mode, uint32_t flags, int conv_m_tiles = 0) {
  if (flags & F_HEAD_FINAL) return 128;   // the head tail needs a whole 128-channel row in one tile
  if (conv_m_tiles > 0) return (N == 256 && (conv_m_tiles + 1) / 2 >= 4 * (num_sms() / 2)) ? 256 : 128;
  // 128x256 tiles for the specialised epilogues (every ViT projection): half the A traffic per FLOP of 128x128
  if (N % 256 == 0 && pick_epi(mode, flags) != EPI_GENERIC) return 256;
  if (N % 128 == 0) return 128;
  if (N % 64 == 0) return 64;
  return (N > 128) ? 128 : 64;            // N % 32 == 0: the last tile is partly empty
}

// 0: 1-CTA kernels, 1: CTA-pair kernels (cluster of two, B tile multicast) whenever BLOCK_N >= 128, 2 (default): pair
// kernels from kPairMinKb k-blocks of 64 on, 1-CTA kernels for the shortest reductions (K = 96 / 192 of the DPT
// re-assembly), whose time goes to the epilogue rather than to operand traffic.
static int g_impl = 2;
constexpr int kPairMinKb = 4;
static bool use_pair(int bn, int num_kb) { return bn >= 128 && (g_impl == 1 || (g_impl == 2 && num_kb >= kPairMinKb)); }

// 0: register-store epilogues everywhere (the bit-identical A/B reference), 1 (default): the specialised epilogues on
// 128x256 tiles stage their output in shared memory and write it by TMA store / TMA reduce-add, when TMA can address it
static int g_store = 1;
// 0: the 3x3 convolutions on the register-store EPI_GENERIC kernels with 128-wide tiles (the bit-identical A/B
// reference), 1 (default): Cout 256 / 128 convs on conv_kernel, with the staged TMA epilogue, when TMA can address every
// tensor the epilogue touches
static int g_conv_store = 1;

static int grid_for(bool pair, int m_tiles, int n_tiles) {
  if (pair) {
    const int items = ((m_tiles + 1) / 2) * n_tiles;
    const int max_clusters = num_sms() / 2;
    return 2 * (items < max_clusters ? items : max_clusters);
  }
  const int items = m_tiles * n_tiles;
  return items < num_sms() ? items : num_sms();
}

static const char* prof_tag(const Params& p, int bn, bool pair) {
  return (p.mode == 1) ? ((p.flags & F_HEAD_FINAL) ? (pair ? "conv3x3_head_tail_2cta" : "conv3x3_head_tail")
                                                   : (pair ? "conv3x3_wgmma_2cta" : "conv3x3_wgmma"))
                       : (bn == 256 ? (pair ? "gemm_wgmma_2cta_bn256" : "gemm_wgmma_bn256")
                                    : (pair ? "gemm_wgmma_2cta_bn128" : (bn == 128 ? "gemm_wgmma_bn128" : "gemm_wgmma_bn64")));
}

template <int BN, int EPI, bool PAIR, bool TMA_STORE = false>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const Params& p, int m_tiles, int n_tiles,
                  cudaStream_t st) {
  constexpr int kSmem = Cfg<BN, TMA_STORE>::kSmemBytes;
  static unsigned long long attr_devices = 0;
  if (first_launch_on_this_device(attr_devices))
    D3R_CUDA(cudaFuncSetAttribute(gemm_kernel<BN, EPI, PAIR, TMA_STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  const int grid = grid_for(PAIR, m_tiles, n_tiles);
  char detail[96];
  snprintf(detail, sizeof(detail), "M=%d N=%d K=%d flags=0x%x mode=%d epi=%d", p.M, p.N, p.K, (unsigned)p.flags, p.mode, EPI);
  prof::Scope scope(prof_tag(p, BN, PAIR), st, 2.0 * double(p.M) * double(p.N) * double(p.K), 0.0, 1, detail);
  D3R_CUDA(pdl::launch_clustered(gemm_kernel<BN, EPI, PAIR, TMA_STORE>, dim3(grid), dim3(kNumThreads), size_t(kSmem), st, PAIR ? 2 : 1,
                                 ta, tb, to, p));
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}

// conv_kernel: profiled under the conv tags with epi=0, like the EPI_GENERIC launches it stands in for
template <int BN, bool PAIR>
static int launch_conv(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const ConvMaps& cm, const Params& p,
                       int m_tiles, int n_tiles, cudaStream_t st) {
  constexpr int kSmem = Cfg<BN, true>::kSmemBytes;
  static unsigned long long attr_devices = 0;
  if (first_launch_on_this_device(attr_devices))
    D3R_CUDA(cudaFuncSetAttribute(conv_kernel<BN, PAIR>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  const int grid = grid_for(PAIR, m_tiles, n_tiles);
  char detail[96];
  snprintf(detail, sizeof(detail), "M=%d N=%d K=%d flags=0x%x mode=%d epi=%d", p.M, p.N, p.K, (unsigned)p.flags, p.mode, EPI_GENERIC);
  prof::Scope scope(prof_tag(p, BN, PAIR), st, 2.0 * double(p.M) * double(p.N) * double(p.K), 0.0, 1, detail);
  D3R_CUDA(pdl::launch_clustered(conv_kernel<BN, PAIR>, dim3(grid), dim3(kNumThreads), size_t(kSmem), st, PAIR ? 2 : 1, ta, tb, to, cm, p));
  D3R_LAUNCH_CHECK();
  return D3R_OK;
}

// `to` != nullptr: the output tensor map of the TMA-store epilogue (BLOCK_N 256, specialised epilogue).  The
// register-store kernels do not read their output map; they are passed tb in its place.
template <int BN, bool PAIR>
static int dispatch_epi(int epi, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* to, const Params& p, int m_tiles,
                        int n_tiles, cudaStream_t st) {
  if constexpr (BN == 256) {
    if (to) {
      switch (epi) {
        case EPI_RESID: return launch<BN, EPI_RESID, PAIR, true>(ta, tb, *to, p, m_tiles, n_tiles, st);
        case EPI_ACT: return launch<BN, EPI_ACT, PAIR, true>(ta, tb, *to, p, m_tiles, n_tiles, st);
        case EPI_ROPE: return launch<BN, EPI_ROPE, PAIR, true>(ta, tb, *to, p, m_tiles, n_tiles, st);
      }
    }
  }
  switch (epi) {
    case EPI_RESID: return launch<BN, EPI_RESID, PAIR>(ta, tb, tb, p, m_tiles, n_tiles, st);
    case EPI_ACT: return launch<BN, EPI_ACT, PAIR>(ta, tb, tb, p, m_tiles, n_tiles, st);
    case EPI_ROPE: return launch<BN, EPI_ROPE, PAIR>(ta, tb, tb, p, m_tiles, n_tiles, st);
  }
  if constexpr (BN == 128) return launch<128, EPI_GENERIC, PAIR>(ta, tb, tb, p, m_tiles, n_tiles, st);
  set_error("no BLOCK_N %d kernel for the generic epilogue", BN);
  return D3R_ERR_INVALID;
}

static int dispatch(int bn, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* to, const Params& p, int m_tiles,
                    cudaStream_t st) {
  const int n_tiles = (p.N + bn - 1) / bn;
  // epilogue specialisations exist for BLOCK_N 128 and 256 (every hot projection of the two ViTs has N % 256 == 0)
  const int epi = (bn >= 128) ? pick_epi(p.mode, p.flags) : EPI_GENERIC;
  const bool pair = use_pair(bn, p.num_kb);
  switch (bn) {
    case 256: return pair ? dispatch_epi<256, true>(epi, ta, tb, to, p, m_tiles, n_tiles, st) : dispatch_epi<256, false>(epi, ta, tb, to, p, m_tiles, n_tiles, st);
    case 128: return pair ? dispatch_epi<128, true>(epi, ta, tb, nullptr, p, m_tiles, n_tiles, st) : dispatch_epi<128, false>(epi, ta, tb, nullptr, p, m_tiles, n_tiles, st);
    case 64: return launch<64, EPI_GENERIC, false>(ta, tb, tb, p, m_tiles, n_tiles, st);
  }
  set_error("unsupported BLOCK_N %d", bn);
  return D3R_ERR_INVALID;
}

// B operand: [N][taps][Kc] bf16, K-major
static int make_tmap_b(CUtensorMap* m, const void* B, int N, int taps, int Kc, int bn, int num_kb, const char* op) {
  cuuint64_t dims[3] = {(cuuint64_t)Kc, (cuuint64_t)taps, (cuuint64_t)N};
  cuuint64_t str[2] = {(cuuint64_t)Kc * 2, (cuuint64_t)taps * Kc * 2};
  cuuint32_t box[3] = {(cuuint32_t)BLOCK_K, 1, (cuuint32_t)(use_pair(bn, num_kb) ? bn / 2 : bn)};   // each CTA of a pair stages half of B
  return encode_tensor_map(m, B, 3, dims, str, box, op);
}

int gemm_bf16(const void* A, long long lda, const void* B, Params p, cudaStream_t st) {
  D3R_CHECK_ARG(A && B, "gemm: null operand");
  D3R_CHECK_ARG(p.M > 0 && p.N > 0 && p.K > 0, "gemm: bad shape %d %d %d", p.M, p.N, p.K);
  D3R_CHECK_ARG(p.N % 32 == 0, "gemm: N=%d must be a multiple of 32", p.N);
  D3R_CHECK_ARG(p.K % 8 == 0 && lda % 8 == 0, "gemm: K=%d / lda=%lld must be multiples of 8 (16-byte TMA strides)", p.K, lda);
  D3R_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0, "gemm: operands must be 16-byte aligned");
  p.mode = 0;
  p.num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;
  const int bn = pick_block_n(p.N, p.mode, p.flags);
  CUtensorMap ta, tb;
  {
    cuuint64_t dims[2] = {(cuuint64_t)p.K, (cuuint64_t)p.M};
    cuuint64_t str[1] = {(cuuint64_t)lda * 2};
    cuuint32_t box[2] = {(cuuint32_t)BLOCK_K, (cuuint32_t)BLOCK_M};
    int rc = encode_tensor_map(&ta, A, 2, dims, str, box, "gemm");
    if (rc) return rc;
  }
  int rc = make_tmap_b(&tb, B, p.N, 1, p.K, bn, p.num_kb, "gemm");
  if (rc) return rc;
  // TMA-store epilogue: [M, N] output boxes of 64 rows x 128 B; TMA needs a 16-byte aligned base and row stride
  CUtensorMap to;
  const bool f32 = (p.flags & F_RESID_INPLACE) != 0;
  const long long row_bytes = p.ldo * (f32 ? 4 : 2);
  const bool staged = g_store == 1 && bn == 256 && pick_epi(p.mode, p.flags) != EPI_GENERIC && p.ldo >= p.N && row_bytes % 16 == 0 &&
                      (reinterpret_cast<uintptr_t>(p.out) & 15) == 0;
  if (staged) {
    cuuint64_t dims[2] = {(cuuint64_t)p.N, (cuuint64_t)p.M};
    cuuint64_t str[1] = {(cuuint64_t)row_bytes};
    cuuint32_t box[2] = {(cuuint32_t)(f32 ? 32 : 64), 64};
    rc = encode_tensor_map(&to, p.out, 2, dims, str, box, "gemm output", f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
    if (rc) return rc;
  }
  return dispatch(bn, ta, tb, staged ? &to : nullptr, p, (p.M + BLOCK_M - 1) / BLOCK_M, st);
}

// (B,H,W,C) bf16 NHWC as a 4D map (C, W, H, B) with boxes of 64 channels x 64 pixels (bw = min(tile_w, 64) by 64 / bw rows):
// one consumer warpgroup's rows of a conv tile
static int make_tmap_conv_io(CUtensorMap* m, const void* base, int B, int H, int W, int C, int tile_w, const char* op) {
  const int bw = tile_w < 64 ? tile_w : 64;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t str[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)bw, (cuuint32_t)(64 / bw), 1};
  return encode_tensor_map(m, base, 4, dims, str, box, op);
}

static bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

int conv3x3_bf16(const void* x_nhwc, const void* w_packed, int B, int H, int W, int Cin, int Cout, Params p, cudaStream_t st) {
  D3R_CHECK_ARG(x_nhwc && w_packed, "conv3x3: null operand");
  D3R_CHECK_ARG(Cin % 8 == 0 && Cout % 32 == 0, "conv3x3: Cin=%d must be a multiple of 8 and Cout=%d of 32", Cin, Cout);
  p.mode = 1;
  p.M = B * H * W;
  p.N = Cout;
  p.cin_blocks = (Cin + BLOCK_K - 1) / BLOCK_K;
  p.K = 9 * Cin;
  p.num_kb = 9 * p.cin_blocks;
  p.cB = B; p.cH = H; p.cW = W;
  int tw = 16;
  while (tw < W && tw < 128) tw *= 2;
  p.tile_w = tw;
  p.tile_h = BLOCK_M / tw;
  p.tiles_x = (W + p.tile_w - 1) / p.tile_w;
  p.tiles_y = (H + p.tile_h - 1) / p.tile_h;
  p.ldo = Cout;
  const int m_tiles = B * p.tiles_x * p.tiles_y;
  // staged epilogue: Cout 256 / 128 (whole 64-channel boxes), the flags EPI_CONV covers, every tensor 16-byte aligned
  const bool staged = g_conv_store == 1 && (Cout == 256 || Cout == 128) && (p.flags & ~EpiMask<EPI_CONV>::value) == 0 &&
                      aligned16(p.out) && (!(p.flags & F_OUT2_RELU) || aligned16(p.out2)) && (!(p.flags & F_ADD0) || aligned16(p.add0)) &&
                      (!(p.flags & F_ADD1) || aligned16(p.add1));
  const int bn = pick_block_n(p.N, p.mode, p.flags, staged ? m_tiles : 0);
  CUtensorMap ta, tb;
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t str[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)W * Cin * 2, (cuuint64_t)H * W * Cin * 2};
    cuuint32_t box[4] = {(cuuint32_t)BLOCK_K, (cuuint32_t)p.tile_w, (cuuint32_t)p.tile_h, 1};
    int rc = encode_tensor_map(&ta, x_nhwc, 4, dims, str, box, "conv3x3");
    if (rc) return rc;
  }
  int rc = make_tmap_b(&tb, w_packed, Cout, 9, Cin, bn, p.num_kb, "conv3x3");
  if (rc) return rc;
  if (!staged) return dispatch(bn, ta, tb, nullptr, p, m_tiles, st);
  CUtensorMap to;
  ConvMaps cm;
  rc = make_tmap_conv_io(&to, p.out, B, H, W, Cout, p.tile_w, "conv3x3 output");
  if (rc) return rc;
  cm.out2 = cm.add0 = cm.add1 = to;   // maps the flags leave unused stay valid (the kernel prefetches all three)
  const struct { uint32_t flag; const void* base; CUtensorMap* map; const char* op; } io[3] = {
      {F_OUT2_RELU, p.out2, &cm.out2, "conv3x3 out2"}, {F_ADD0, p.add0, &cm.add0, "conv3x3 add0"}, {F_ADD1, p.add1, &cm.add1, "conv3x3 add1"}};
  for (const auto& t : io) {
    if (!(p.flags & t.flag)) continue;
    rc = make_tmap_conv_io(t.map, t.base, B, H, W, Cout, p.tile_w, t.op);
    if (rc) return rc;
  }
  const int n_tiles = Cout / bn;
  const bool pair = use_pair(bn, p.num_kb);
  if (bn == 256) return pair ? launch_conv<256, true>(ta, tb, to, cm, p, m_tiles, n_tiles, st) : launch_conv<256, false>(ta, tb, to, cm, p, m_tiles, n_tiles, st);
  return pair ? launch_conv<128, true>(ta, tb, to, cm, p, m_tiles, n_tiles, st) : launch_conv<128, false>(ta, tb, to, cm, p, m_tiles, n_tiles, st);
}

// rows = input pixels, columns = (ky,kx,co).  The epilogue stores column pairs (co, co + 1), so Cout must be even for a
// pair to stay inside one kernel position.
int conv_transpose_bf16(const void* x_nhwc, const void* w_packed, void* out, const float* bias, int B, int h, int w, int Cin, int Cout,
                        int k, cudaStream_t st) {
  D3R_CHECK_ARG(x_nhwc && w_packed && out, "conv_transpose: null buffer");
  D3R_CHECK_ARG(B > 0 && h > 0 && w > 0 && Cin > 0 && Cout > 0 && k > 0, "conv_transpose: bad shape B=%d h=%d w=%d Cin=%d Cout=%d k=%d", B,
                h, w, Cin, Cout, k);
  D3R_CHECK_ARG(Cin % 8 == 0, "conv_transpose: Cin=%d must be a multiple of 8", Cin);
  D3R_CHECK_ARG(Cout % 2 == 0 && (k * k * Cout) % 32 == 0, "conv_transpose: Cout=%d must be even and k*k*Cout=%d a multiple of 32", Cout,
                k * k * Cout);
  Params p{};
  p.M = B * h * w; p.N = k * k * Cout; p.K = Cin;
  p.flags = F_CONVT | (bias ? F_BIAS : 0);
  p.out = out; p.bias = bias; p.ldo = 0;
  p.tk = k; p.th_in = h; p.tw_in = w; p.tCout = Cout;
  return gemm_bf16(x_nhwc, Cin, w_packed, p, st);
}

int conv3x3_head_tail(const void* x_nhwc, const void* w_packed, const float* bias, const float* w4, const float* b4, float* pts3d,
                      float* conf, int B, int H, int W, int depth_mode, int conf_mode, float conf_min, float conf_max, cudaStream_t st) {
  D3R_CHECK_ARG(x_nhwc && w_packed && w4 && b4 && pts3d, "conv3x3_head_tail: null buffer");
  D3R_CHECK_ARG(B > 0 && H > 0 && W > 0, "conv3x3_head_tail: bad shape B=%d H=%d W=%d", B, H, W);
  D3R_CHECK_ARG(depth_mode >= 0 && depth_mode <= 2, "conv3x3_head_tail: depth_mode %d out of range", depth_mode);
  D3R_CHECK_ARG(conf_mode >= 0 && conf_mode <= 2, "conv3x3_head_tail: conf_mode %d out of range", conf_mode);
  D3R_CHECK_ARG(conf_mode == 0 || conf, "conv3x3_head_tail: conf_mode %d without a conf buffer", conf_mode);
  Params p{};
  p.flags = F_HEAD_FINAL | (bias ? F_BIAS : 0);
  p.bias = bias;
  p.w4 = w4; p.b4 = b4;
  p.pts3d = pts3d; p.conf = conf;
  p.depth_mode = depth_mode; p.conf_mode = conf_mode;
  p.conf_min = conf_min; p.conf_max = conf_max;
  return conv3x3_bf16(x_nhwc, w_packed, B, H, W, 128, 128, p, st);
}

}  // namespace gemm
}  // namespace d3r

// ---- building blocks exported through the C ABI (used by the unit tests and by forward.cu) ----
using namespace d3r;

extern "C" void d3r_set_gemm_impl(int32_t impl) { gemm::g_impl = impl; }
extern "C" void d3r_set_gemm_store(int32_t store) { gemm::g_store = store; }
extern "C" void d3r_set_conv_store(int32_t store) { gemm::g_conv_store = store; }

extern "C" int d3r_gemm_bf16(const void* A, const void* B, void* out, const float* bias, const void* add0, void* out2,
                             int32_t M, int32_t N, int32_t K, int64_t ldo, uint32_t flags, const float* rope_cos,
                             const float* rope_sin, int32_t rope_cols, int32_t tokens_per_img, int32_t grid_w, void* stream) {
  gemm::Params p{};
  p.M = M; p.N = N; p.K = K;
  p.flags = flags;
  p.out = out; p.out2 = out2; p.add0 = add0; p.bias = bias; p.ldo = ldo;
  p.rope_cos = rope_cos; p.rope_sin = rope_sin; p.rope_cols = rope_cols; p.tokens_per_img = tokens_per_img; p.grid_w = grid_w;
  D3R_CHECK_ARG(!(flags & gemm::F_BIAS) || bias, "gemm: F_BIAS without bias");
  D3R_CHECK_ARG(!(flags & gemm::F_ROPE) || (rope_cos && rope_sin && tokens_per_img > 0 && grid_w > 0), "gemm: F_ROPE without tables");
  D3R_CHECK_ARG(!(flags & (gemm::F_CONVT | gemm::F_HEAD_FINAL)),
                "gemm: F_CONVT / F_HEAD_FINAL have their own entry points, d3r_conv_transpose_bf16 / d3r_conv3x3_head_tail");
  return gemm::gemm_bf16(A, K, B, p, (cudaStream_t)stream);
}

extern "C" int d3r_conv3x3_bf16(const void* x_nhwc, const void* w_packed, void* out, const float* bias, const void* add0,
                                const void* add1, void* out2, int32_t B, int32_t H, int32_t W, int32_t Cin, int32_t Cout,
                                uint32_t flags, void* stream) {
  gemm::Params p{};
  p.flags = flags;
  p.out = out; p.out2 = out2; p.add0 = add0; p.add1 = add1; p.bias = bias;
  D3R_CHECK_ARG(!(flags & (gemm::F_CONVT | gemm::F_HEAD_FINAL | gemm::F_ROPE)), "conv3x3: unsupported flag");
  return gemm::conv3x3_bf16(x_nhwc, w_packed, B, H, W, Cin, Cout, p, (cudaStream_t)stream);
}

extern "C" int d3r_conv_transpose_bf16(const void* x_nhwc, const void* w_packed, void* out, const float* bias, int32_t B, int32_t h,
                                       int32_t w, int32_t Cin, int32_t Cout, int32_t k, void* stream) {
  return gemm::conv_transpose_bf16(x_nhwc, w_packed, out, bias, B, h, w, Cin, Cout, k, (cudaStream_t)stream);
}

extern "C" int d3r_conv3x3_head_tail(const void* x_nhwc, const void* w_packed, const float* bias, const float* w4, const float* b4,
                                     float* pts3d, float* conf, int32_t B, int32_t H, int32_t W, int32_t depth_mode, int32_t conf_mode,
                                     float conf_min, float conf_max, void* stream) {
  return gemm::conv3x3_head_tail(x_nhwc, w_packed, bias, w4, b4, pts3d, conf, B, H, W, depth_mode, conf_mode, conf_min, conf_max,
                                 (cudaStream_t)stream);
}
