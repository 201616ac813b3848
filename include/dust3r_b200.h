/*
 * dust3r_b200 — C ABI of the H100-native DUSt3R hot paths (sm_90a).
 *
 * The reference (naver/dust3r) has no FFI/plugin registry; its only native entry point is the
 * pybind function `curope.rope_2d` (croco/models/curope/curope.cpp:49-69).  Everything else on
 * the two hot paths is Python calling torch.  This header is therefore the boundary a
 * maintainer binds with ctypes (see INTEGRATION.md): plain pointers + sizes + a cudaStream_t,
 * int return codes, no torch / ATen / Python types.
 *
 * Conventions
 *   - every pointer marked `dev` is a CUDA device pointer owned by the caller (PyTorch owns all
 *     memory; the library never allocates caller-visible memory);
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream);
 *   - return value 0 = success, negative = error; d3r_last_error() gives the message of the
 *     last failure on the calling thread;
 *   - calls are asynchronous w.r.t. the host unless stated; thread-safe for distinct streams.
 */
#ifndef DUST3R_B200_H_
#define DUST3R_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define D3R_OK 0
#define D3R_ERR_INVALID (-1)   /* bad argument / unsupported shape   */
#define D3R_ERR_CUDA (-2)      /* CUDA runtime / driver error        */
#define D3R_ERR_UNSUPPORTED_DEVICE (-3)

const char* d3r_last_error(void);
/* ABI version of this header; bumped on any signature change. */
int d3r_abi_version(void);
/* 0 when the current device is sm_90 (H100); D3R_ERR_UNSUPPORTED_DEVICE otherwise. */
int d3r_check_device(void);

/* Launch accounting / profiling aid: number of kernels this library launched since the last reset;
 * with d3r_prof_enable(1) every launch is bracketed by CUDA events on its stream and
 * d3r_prof_report() returns a JSON object {tag: {count, ms, flops, bytes}} (returns length, -1 if
 * the buffer is too small). */
long long d3r_launch_count(void);
void d3r_launch_count_reset(void);
void d3r_prof_enable(int on);
int d3r_prof_report(char* buf, int cap);
/* every recorded launch in order: JSON list [{tag, detail, ms, flops, bytes}] (length, or -1 if it does not fit) */
int d3r_prof_dump(char* buf, int cap);

/* ------------------------------------------------------------------------------------------
 * Path 2 — global alignment (replaces the body of global_alignment_iter(),
 * dust3r/cloud_opt/base_opt.py:352-366: zero_grad + PointCloudOptimizer.forward
 * (optimizer.py:188-201) or BasePCOptimizer.forward (base_opt.py:246-273) + loss.backward() +
 * torch.optim.Adam.step(), for every iteration of global_alignment_loop, base_opt.py:326-349).
 *
 * One launch per iteration: unproject depth -> 3D, confidence-weighted pairwise distance,
 * analytic backward, Adam on the per-pixel log-depths; the last CTA folds the per-edge /
 * per-image partial sums into pose / focal / principal-point / pairwise-pose gradients, applies
 * Adam to them and refreshes the transforms for the next launch.
 * ------------------------------------------------------------------------------------------ */

/* Small parameters live in ONE float buffer `small` (and two more of the same layout for Adam's
 * exp_avg / exp_avg_sq, plus a uint8 buffer of trainable flags):
 *   [ im_poses n*7 | im_focals n*2 | im_pp n*2 | pw_poses E*8 | pw_adaptors E*2 ]
 * im_poses / pw_poses rows are [qx,qy,qz,qw, tx,ty,tz(, log_scale)] exactly as
 * optimizer.py:30 / base_opt.py:90 store them; im_focals holds focal_break*log(f) twice when the
 * model has a single focal (fx == fy, tied). */
typedef struct d3r_align_desc {
  int32_t n_imgs;          /* n                                                             */
  int32_t n_edges;         /* E (directed edges, base_opt.py:61)                            */
  int32_t n_entries;       /* 2*E : one entry per (edge, side)                              */
  int32_t n_chunks;        /* total CTAs = sum_i ceil(P_i / chunk_px)                       */
  int32_t max_deg;         /* max entries incident to one image                             */
  int32_t max_chunks;      /* max CTAs of one image                                         */
  int32_t chunk_px;        /* pixels per CTA, 1..d3r_align_chunk_pixels() (host picks it so
                              the grid is a whole number of waves)                          */
  int32_t dist_l2;         /* 0: l1_dist, 1: l2_dist (commons.py:62-70)                     */
  int32_t norm_pw_scale;   /* base_opt.py:86,178-184                                        */
  int32_t tied_focal;      /* 1: one focal per image (fx==fy), 0: fx_and_fy                 */
  int32_t eval_only;       /* 1: only write the loss (net.forward()), no parameter update   */
  float base_scale;        /* base_opt.py:49                                                */
  float pw_break;          /* base_opt.py:51                                                */
  float focal_break;       /* optimizer.py:22 / modular_optimizer.py:24 (focal_brake)       */
  float adam_eps;          /* 1e-8                                                          */
  float beta1, beta2;      /* (0.9, 0.9) base_opt.py:337                                    */

  /* per image (dev) */
  const int32_t* img_hw;        /* [n][2] = H, W                                            */
  const int64_t* img_pix_off;   /* [n+1] offset of image i's pixels in logd / adam buffers  */
  const int32_t* img_ent_ptr;   /* [n+1] CSR into the entry arrays                          */
  const int32_t* img_chunk_ptr; /* [n+1] first CTA index of image i                         */
  /* per CTA (dev) */
  const int32_t* chunk_img;     /* [n_chunks] image handled by CTA c                        */
  /* per entry, CSR order (dev) */
  const int32_t* ent_edge;      /* [2E] edge id                                             */
  const int64_t* ent_obs_off;   /* [2E] offset (in float4) of the entry's observations      */
  const float*   ent_coef;      /* [2E] loss coefficient: 1/total_area (stacked) or 1/(P*E) */
  const int32_t* edge_ent;      /* [E][2] entry index of (edge, side i) and (edge, side j)  */
  /* observations (dev): float4 = (pred.x, pred.y, pred.z, weight) per pixel per entry.
   * 32*E*P bytes in total = the read-once traffic of SURVEY §8d.                          */
  const void* obs;

  /* trainable state (dev) */
  float* logd;                  /* [sum P_i] log-depth, optimizer.py:29                     */
  float* logd_m;                /* Adam exp_avg                                             */
  float* logd_v;                /* Adam exp_avg_sq                                          */
  float* small;                 /* layout above                                             */
  float* small_m;
  float* small_v;
  const uint8_t* small_trainable; /* same layout, 1 = requires_grad                         */

  /* derived per-iteration state + scratch (dev), sizes from d3r_align_workspace_floats()  */
  float* workspace;
  /* [niter_total][4] = lr, lr/bias_correction1, sqrt(bias_correction2), 0 for every step   */
  const float* sched;
  float* loss_out;              /* [niter_total] loss of every iteration                    */
  int32_t* counters;            /* [n + 2] zero-initialised by the caller once              */
  /* `workspace` must be zero-initialised by the caller once as well (accumulators live there).  */

  /* ---- streaming kernel (csrc/align_stream.cu), used when every image has P % 4 == 0 and a pixel stride
   * that is a multiple of 4 (always true for DUSt3R inputs: H, W are multiples of the 16-pixel patch).
   * stream_kernel = 1 selects it; obs then holds the slot-interleaved layout written by
   * d3r_align_pack_entries with stream_layout = 1 (same 16 bytes per observation):
   *   per entry: slots of 64 pixels = [32 x (xA,xB,yA,yB)] [32 x (zA,zB,wA,wB)] for the 32 pixel pairs
   *   (A,B) = (2j, 2j+1) of the slot, the loss coefficient folded into w; every image's slab is padded to
   *   whole slots with w = 0.
   * The pixel range of every image is cut into work items of <= ppt slots; persistent warp w owns items
   * [warp_item_ptr[w], warp_item_ptr[w+1]).                                                           */
  int32_t stream_kernel;
  int32_t stream_grid;          /* CTAs of the persistent grid                                       */
  int32_t stream_ppt;           /* slots (64 pixels) per work item, 3                                 */
  int32_t stream_window;        /* entries whose partial sums a warp keeps in shared memory            */
  int32_t n_items;
  int32_t reserved0;
  const void* items;            /* [n_items] d3r_align_item                                            */
  const int32_t* warp_item_ptr; /* [stream_grid * 8 + 1]                                               */
  /* Optional second traversal of the same items in REVERSE global order (items_rev[k] = items[n_items-1-k],
   * with its own warp split).  When set, odd iterations walk it: what an iteration streamed last is what
   * the next one streams first, so the tail of every pass is still resident in the 126 MB L2 (observations
   * are constants of the problem).  NULL = every iteration walks `items`.                              */
  const void* items_rev;
  const int32_t* warp_item_ptr_rev;
} d3r_align_desc;

/* One work item of the streaming kernel: `nslots` consecutive 64-pixel slots of image `img`. */
typedef struct d3r_align_item {
  int32_t img, slot0, nslots, npx;     /* npx: valid pixels of the item (multiple of 4)               */
  int32_t e0, deg, W, u0;              /* first entry / number of entries of the image; width; column of the first pixel */
  int32_t v0;                          /* row of the first pixel                                      */
  float inv_w;                         /* 1 / W                                                       */
  int64_t pix0;                        /* img_pix_off[img] + 64 * slot0: index into logd / adam moments */
  int64_t obs0;                        /* 16-byte units: first entry's slab of the image + 64 * slot0   */
  int32_t slab_units;                  /* 16-byte units per entry slab of this image (64 * slots)      */
  int32_t reserved;
} d3r_align_item;

/* sizeof(d3r_align_desc) / sizeof(d3r_align_item) as compiled into the library (binding self-check). */
int d3r_sizeof_align_desc(void);
int d3r_sizeof_align_item(void);
/* Maximum pixels one CTA of the alignment kernel can take (compile-time constant of the library). */
int d3r_align_chunk_pixels(void);
/* Number of floats of `workspace` needed for a problem of this size. */
int64_t d3r_align_workspace_floats(int32_t n_imgs, int32_t n_edges);
/* Computes the transforms used by the first iteration from `small` (call once after the
 * parameters are (re)initialised or modified from the host). */
int d3r_align_prepare(const d3r_align_desc* desc, void* stream);
/* Runs iterations [it_begin, it_end) (indices into sched / loss_out).  Asynchronous. */
int d3r_align_run(const d3r_align_desc* desc, int32_t it_begin, int32_t it_end, void* stream);
/* One iteration as two launches, so that a caller can combine the cross-CTA sums of several GPUs in between:
 *   d3r_align_pixel_pass(desc, it)   the streaming kernel's per-pixel work over desc's items (unprojection, residuals,
 *                                    dL/dlog-depth, the depth Adam step) -- nothing is launched when n_items == 0;
 *   all-reduce(SUM) of the int64 block that d3r_align_reduce_block locates in `workspace` (optional: one GPU needs none);
 *   d3r_align_small_step(desc, it)   the small-parameter step of d3r_align_run's last CTA on the (reduced) sums: loss_out[it],
 *                                    Adam on `small`, the derived transforms; with desc->eval_only only loss_out[it].
 * Streaming kernel only (stream_kernel = 1).  On one GPU the pair gives the same bits as d3r_align_run(desc, it, it + 1).
 * Every GPU runs the small step on the same reduced block and so computes the same `small`; each GPU's pixel pass updates
 * only the log-depths of its own items' images.  The block is [ent_acc | img_acc | overflow word]: the fixed-point sums
 * (integers, so the all-reduce is exact and order-independent) and a word the pixel pass makes non-zero when a partial sum
 * left the range or met a NaN / Inf, which the small step turns into the overflow flag.  Asynchronous. */
int d3r_align_pixel_pass(const d3r_align_desc* desc, int32_t it, void* stream);
int d3r_align_small_step(const d3r_align_desc* desc, int32_t it, void* stream);
/* *offset_floats: where the all-reduce block starts in `workspace` (in floats, 16-byte aligned); *n_words: its length in int64. */
int d3r_align_reduce_block(int32_t n_imgs, int32_t n_edges, int64_t* offset_floats, int64_t* n_words);
/* d3r_align_loss_grad (below) as two launches around the same all-reduce of the d3r_align_reduce_block block:
 *   d3r_align_grad_pixel_pass(desc, logd_grad)   the gradient launch's per-pixel work over desc's items: dL/dlog-depth of
 *                                                their pixels to logd_grad (other pixels are not written: pass a zeroed
 *                                                buffer), the sums, and the overflow word -- nothing is launched when
 *                                                n_items == 0;
 *   all-reduce(SUM) of the block (optional: one GPU needs none);
 *   d3r_align_grad_small_step(desc, small_grad, entry_loss)   the gradient launch's last-CTA step on the (reduced) sums:
 *                                                loss -> desc->loss_out[0], small_grad, entry_loss (may be NULL).
 * Streaming kernel only (stream_kernel = 1).  The contract is d3r_align_loss_grad's: no parameter or Adam moment is touched
 * (logd_m, logd_v, small_m, small_v, small_trainable and sched may be NULL), the accumulators and the overflow word are left
 * cleared, the small step sets the overflow flag, and when it is set loss_out[0], every element of small_grad and of
 * entry_loss are NaN.  On one GPU the pair gives the bits of d3r_align_loss_grad; on several, each GPU's pixel pass writes
 * the log-depth gradients of its own items' images, and every GPU's small step computes the same loss and small_grad.
 * Asynchronous. */
int d3r_align_grad_pixel_pass(const d3r_align_desc* desc, float* logd_grad, void* stream);
int d3r_align_grad_small_step(const d3r_align_desc* desc, float* small_grad, float* entry_loss, void* stream);
/* Objective and its gradient at the current parameters (net.forward() + loss.backward()): one launch of the pixel kernel
 * the descriptor selects + the last-CTA small step.  Updates no parameter or Adam moment; reads neither sched nor the moments
 * (logd_m, logd_v, small_m, small_v, small_trainable and sched may be NULL).  Call d3r_align_prepare first when `small` changed.
 * loss -> desc->loss_out[0] (bit-identical to an eval_only run).  logd_grad [sum stride_i]: dL/dlog-depth (padding pixels are
 * not written: pass a zeroed buffer).  small_grad [11n+10E]: dL/d(raw parameter) in the `small` layout, complete: log-scale
 * mean coupling and adaptor mean removal folded in; with tied focals both focal slots hold the full dL/dfocal.  Gradients of
 * every parameter, whatever small_trainable says.  entry_loss (may be NULL) [E][2]: coefficient-weighted loss of (edge, side).
 * Sets the overflow flag like a run; leaves the accumulators cleared, so a following d3r_align_run is unaffected.  When the
 * flag is set (a NaN / Inf observation, or a sum out of the fixed-point range), loss_out[0], every element of small_grad and
 * of entry_loss are NaN, so that an out-of-range scene never returns a finite objective without a host check. */
int d3r_align_loss_grad(const d3r_align_desc* desc, float* logd_grad, float* small_grad, float* entry_loss, void* stream);
/* Cross-CTA sums use order-independent 2^40 fixed-point integer atomics (bit-reproducible).  *host_out = 1 when a
 * partial sum (|x| >= 2^18) or a total (|x| >= 2^22) left the supported range (unreasonably scaled scene, NaN / Inf input)
 * since iteration 0 of the current d3r_align_run batch (or of the split iterations), or during the last d3r_align_loss_grad
 * (or d3r_align_grad_pixel_pass + d3r_align_grad_small_step).  Every iteration from the one
 * that set it writes NaN to loss_out (eval_only runs included). */
int d3r_align_overflow_flag(const d3r_align_desc* desc, int32_t* host_out, void* stream);
/* World-frame pointmaps X[i] = R_i * unproject(depth_i) + T_i for every image
 * (PointCloudOptimizer.depth_to_pts3d, optimizer.py:170-180).  out: [sum P_i][3] float. */
int d3r_align_pts3d(const d3r_align_desc* desc, float* out_dev, void* stream);
/* Debug aid: when dev_buf != NULL every CTA of the next alignment launches writes 4 uint64 %globaltimer stamps
 * (start, end of pixel phase, end/exit, end of small-parameter step) at dev_buf[4*cta]. */
int d3r_align_set_debug(void* dev_buf);

/* Packs EVERY entry's observations in one launch, straight from the (device-resident) output of the forward:
 * replaces the ParameterStack copies + conf_trf of optimizer.py:50-57 / base_opt.py:72-75.  `table` (dev) has one
 * row per entry; the confidence transform (commons.py:73-80: D3R_CONF_ID / LOG / SQRT / M1) is applied on the fly.
 * stream_layout = 0: plain float4 (x, y, z, w) rows; 1: the slot-interleaved layout of the streaming kernel, the
 * loss coefficient folded into w and slabs padded to whole 64-pixel slots with zeros. */
#define D3R_CONF_ID 0
#define D3R_CONF_LOG 1
#define D3R_CONF_SQRT 2
#define D3R_CONF_M1 3
typedef struct d3r_pack_entry {
  const float* pts;        /* dev: (area, 3) pointmap of the entry                                       */
  const float* conf;       /* dev: (area) raw confidence                                                  */
  int64_t obs_off;         /* float4 units: where the entry's slab starts in obs                          */
  int32_t area;            /* pixels of the entry                                                         */
  float coef;              /* loss coefficient of the entry (folded into w when stream_layout = 1)        */
} d3r_pack_entry;
int d3r_sizeof_pack_entry(void);
/* Compile-time constants of the streaming kernel the host needs to build the work-item table: slots (64 pixels) per
 * item, persistent warps per CTA, and the largest entry window for which two CTAs still fit one SM. */
int d3r_align_stream_slots_per_item(void);
int d3r_align_stream_warps_per_cta(void);
int d3r_align_stream_max_window(void);
int d3r_align_pack_entries(const d3r_pack_entry* table_dev, int32_t n_entries, int32_t max_area, int32_t conf_mode,
                           int32_t stream_layout, void* obs_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Path 1 building blocks — exported so the parity tests can exercise each kernel in isolation.
 * Integrators use d3r_encode_images / d3r_decode_pairs below; these are the ops they are composed of.
 * ------------------------------------------------------------------------------------------ */

/* epilogue flags of d3r_gemm_bf16 / d3r_conv3x3_bf16 */
#define D3R_F_BIAS          (1u << 0)
#define D3R_F_GELU          (1u << 1)   /* exact erf GELU (croco/models/blocks.py Mlp act_layer=nn.GELU) */
#define D3R_F_RELU          (1u << 2)
#define D3R_F_OUT_F32       (1u << 3)
#define D3R_F_RESID_INPLACE (1u << 4)   /* out(f32) += result : residual stream update                   */
#define D3R_F_ADD0          (1u << 5)
#define D3R_F_ADD1          (1u << 6)
#define D3R_F_OUT2_RELU     (1u << 7)
#define D3R_F_ROPE          (1u << 8)   /* 2D RoPE on columns < rope_cols; replaces curope.rope_2d        */
#define D3R_F_OUT2_BF16     (1u << 11)

/* out[M,N] = epilogue(A[M,K] * B[N,K]^T); A, B bf16 row-major (nn.Linear weight layout), wgmma.
 * N % 32 == 0, K % 8 == 0.  With D3R_F_ROPE: rope_cos/sin are [max_pos][16] fp32 tables
 * (angle = pos * base^(-k/16), croco/models/curope/kernels.cu:41-52), rows are tokens of images of
 * `tokens_per_img` tokens laid out row-major on a grid `grid_w` wide. */
int d3r_gemm_bf16(const void* A_dev, const void* B_dev, void* out_dev, const float* bias_dev, const void* add0_dev,
                  void* out2_dev, int32_t M, int32_t N, int32_t K, int64_t ldo, uint32_t flags,
                  const float* rope_cos_dev, const float* rope_sin_dev, int32_t rope_cols, int32_t tokens_per_img,
                  int32_t grid_w, void* stream);

/* 3x3 stride-1 pad-1 convolution as implicit GEMM on wgmma.  x: (B,H,W,Cin) bf16 NHWC;
 * w_packed: [Cout][ky*3+kx][Cin] bf16; out/add0/add1/out2: (B,H,W,Cout) bf16 NHWC.
 * (croco/models/dpt_block.py ResidualConvUnit_custom / layer_rn / head convs) */
int d3r_conv3x3_bf16(const void* x_nhwc_dev, const void* w_packed_dev, void* out_dev, const float* bias_dev,
                     const void* add0_dev, const void* add1_dev, void* out2_dev, int32_t B, int32_t H, int32_t W,
                     int32_t Cin, int32_t Cout, uint32_t flags, void* stream);

/* softmax(q k^T * scale) v, head dim 64, bf16 in/out, fp32 softmax (croco/models/blocks.py:94-112,
 * 146-169).  q rows at (b*Nq+i)*ldq + h*64, k/v rows at (b*Nk+j)*ld{k,v} + h*64, out like q. */
int d3r_attention_hd64(const void* q_dev, int64_t ldq, const void* k_dev, int64_t ldk, const void* v_dev, int64_t ldv,
                       void* out_dev, int64_t ldo, int32_t B, int32_t heads, int32_t Nq, int32_t Nk, float scale,
                       void* stream);

/* ConvTranspose2d with kernel == stride == k (dpt_block.py act_postprocess 0 / 1) as a GEMM whose epilogue scatters each
 * input pixel's k x k x Cout block: x (B,h,w,Cin) bf16 NHWC; w_packed [(ky*k+kx)*Cout + co][Cin] bf16 (the torch weight
 * (Cin,Cout,k,k) permuted to (ky,kx,co,ci)); bias [Cout] fp32 or NULL; out (B,h*k,w*k,Cout) bf16 NHWC.
 * Cin % 8 == 0, Cout even, k*k*Cout % 32 == 0. */
int d3r_conv_transpose_bf16(const void* x_nhwc_dev, const void* w_packed_dev, void* out_dev, const float* bias_dev, int32_t B,
                            int32_t h, int32_t w, int32_t Cin, int32_t Cout, int32_t k, void* stream);

/* DPT head tail (dpt_head.py head.2 .. head.4 + postprocess.py), fused into one conv's epilogue: conv3x3 128->128 (+ bias, may
 * be NULL) -> ReLU -> 1x1 conv to 4 channels (w4 [4][128], b4 [4] fp32; rows past the model's channels zero) -> pointmap
 * postprocess.  x (B,H,W,128) bf16 NHWC, w_packed [128][9][128] bf16; pts3d (B,H,W,3) fp32; conf (B,H,W) fp32, written only
 * when conf_mode != 0.  depth_mode 0 linear, 1 square, 2 exp; conf_mode 0 none, 1 exp, 2 sigmoid, in [conf_min, conf_max]. */
int d3r_conv3x3_head_tail(const void* x_nhwc_dev, const void* w_packed_dev, const float* bias_dev, const float* w4_dev,
                          const float* b4_dev, float* pts3d_dev, float* conf_dev, int32_t B, int32_t H, int32_t W, int32_t depth_mode,
                          int32_t conf_mode, float conf_min, float conf_max, void* stream);

/* LayerNorm of fp32 rows to bf16 (nn.LayerNorm of the ViT blocks): x [M][C] fp32, g / b [C] fp32, out [M][C] bf16.
 * C % 4 == 0, C <= 2048; x, g, b 16-byte aligned. */
int d3r_layernorm_bf16(const float* x_dev, const float* g_dev, const float* b_dev, void* out_dev, int32_t M, int32_t C, float eps,
                       void* stream);

/* Bilinear x2 upsample, align_corners=True (dpt_block.py F.interpolate), cropped: x (B,H,W,C) bf16 NHWC -> out (B,Ho,Wo,C), the
 * top-left Ho x Wo of the (2H, 2W) upsample.  Ho <= 2H, Wo <= 2W, C/8 a power of two; buffers 16-byte aligned. */
int d3r_upsample2x_bf16(const void* x_dev, void* out_dev, int32_t B, int32_t H, int32_t W, int32_t C, int32_t Ho, int32_t Wo,
                        void* stream);

/* im2col of the 3x3 stride-2 pad-1 conv (act_postprocess 3): x (B,H,W,C) bf16 NHWC -> out [B*Ho*Wo][9][C] with
 * Ho = ceil(H/2), Wo = ceil(W/2), tap = ky*3+kx, zero outside the image.  C % 8 == 0. */
int d3r_im2col_3x3_s2_bf16(const void* x_dev, void* out_dev, int32_t B, int32_t H, int32_t W, int32_t C, void* stream);

/* Patch im2col of the 16x16 patch embedding: img (B,3,H,W) fp32 -> out [B*(H/16)*(W/16)][3*16*16] bf16 (round to nearest
 * even), column c*256 + py*16 + px (the Conv2d weight flatten).  H, W multiples of 16. */
int d3r_patch_im2col16(const float* img_dev, void* out_dev, int32_t B, int32_t H, int32_t W, void* stream);

/* Linear head tail (heads/linear_head.py + postprocess.py): feat [B*gh*gw][nch*256] fp32 (channel-major, then py*16+px)
 * -> pixel shuffle -> pts3d (B,16gh,16gw,3), conf (B,16gh,16gw) fp32 (conf written only when nch == 4 and conf_mode != 0). */
int d3r_linear_head_postprocess(const float* feat_dev, float* pts3d_dev, float* conf_dev, int32_t B, int32_t gh, int32_t gw,
                                int32_t nch, int32_t depth_mode, int32_t conf_mode, float conf_min, float conf_max, void* stream);

/* Selects the GEMM / conv kernel family: 0 = 1-CTA kernels, 1 = CTA-pair kernels (a cluster of two CTAs on two
 * M tiles sharing one multicast B tile), 2 (default) = CTA-pair kernels from 4 k-blocks of 64 on (K >= 256, a fixed
 * threshold), 1-CTA for shorter reductions. */
void d3r_set_gemm_impl(int32_t impl);
/* Selects how the specialised epilogues on 128x256 tiles (bias / GELU / ReLU -> bf16, bias + RoPE -> bf16, fp32 residual
 * update) write their result: 1 (default) = staged in shared memory and written by TMA store, or TMA reduce-add for the
 * residual update, overlapping the next tile's main loop; 0 = every thread stores straight from its accumulator
 * registers (A/B reference, bit-identical).  With 1, an output whose base or row stride (ldo * element size) is not a
 * multiple of 16 bytes takes the register stores. */
void d3r_set_gemm_store(int32_t store);
/* Selects how the 3x3 convolutions with Cout 256 or 128 (d3r_conv3x3_bf16 and the DPT head; not the head tail) run:
 * 1 (default) = 128x256 tiles where the launch has at least 4 waves of work at that width, else 128x128, with the
 * epilogue staged in shared memory (addends loaded into it by TMA) and written by TMA store, overlapping the next tile's
 * main loop; 0 = 128x128 tiles whose threads load the addends and store straight from their accumulator registers (A/B
 * reference, bit-identical).  With 1, a tensor whose base is not 16-byte aligned selects the register stores. */
void d3r_set_conv_store(int32_t store);

/* Selects the attention kernel: 3 (default) = wgmma kernel (64 query rows per warpgroup, 128-key blocks) with P kept in
 * registers (A-from-registers wgmma); 2 = the same dataflow with P through shared memory (A/B reference). */
void d3r_set_attention_impl(int32_t impl);

/* ------------------------------------------------------------------------------------------
 * Scene-level operators either side of the alignment loop (SURVEY section 8f).  Device pointers, fp32.
 * ------------------------------------------------------------------------------------------ */
/* clean_pointcloud (dust3r/cloud_opt/base_opt.py:369-405): conf[i][p] is cut to bad_conf when image i's world point p lands
 * in image j in front of j's surface ((1 - tol) * depth_j) where j is more confident; (i, j) visited in the reference's order
 * (later tests see earlier cuts).  Images are packed back to back: image i = rows [off[i], off[i] + hw[2i] * hw[2i+1]) of
 * pts3d [.][3] (world frame), conf (updated in place) and depth.  K: [n][3][3], cams: [n][4][4] world-to-camera, row-major. */
int d3r_clean_pointcloud(int32_t n_imgs, const int32_t* hw_dev, const int64_t* off_dev, int32_t max_area, const float* pts3d_dev,
                         float* conf_dev, const float* depth_dev, const float* K_dev, const float* cams_dev, float tol,
                         float bad_conf, void* stream);
/* Moments of the weighted Umeyama / Kabsch problems roma.rigid_points_registration solves for
 * dust3r/cloud_opt/init_im_poses.py:66-110, 253-262: per problem b, out[b][17] (fp64) =
 * { sum w | sum w x (3) | sum w y (3) | sum w y x^T (9, row-major) | sum w |x|^2 } over the n_points rows of x, y [B][P][3], w [B][P]. */
int d3r_procrustes_moments(int32_t n_problems, int32_t n_points, const float* x_dev, const float* y_dev, const float* w_dev,
                           double* out_dev, void* stream);
/* estimate_focal_knowing_depth(..., focal_mode='weiszfeld') (dust3r/post_process.py:12-60) without its final clipping:
 * pts3d [B][H][W][3] in the camera frame, pp [B][2] -> focal [B] after `steps` re-weighted iterations. */
int d3r_weiszfeld_focal(int32_t n_maps, int32_t H, int32_t W, const float* pts3d_dev, const float* pp_dev, int32_t steps,
                        float* focal_dev, void* stream);
/* Index of the nearest of `points` [M][3] for every row of `queries` [N][3] (squared Euclidean distance, lowest index on a
 * tie): the two tree queries of find_reciprocal_matches (dust3r/utils/geometry.py:345-361), brute force on the GPU. */
int d3r_nearest_neighbours(int32_t n_queries, int32_t n_points, const float* queries_dev, const float* points_dev, int32_t* nn_dev,
                           void* stream);
/* Per-image pixel work of load_images (dust3r/utils/image.py:62-71 `_resize_pil_image`, :101-124 crop + ImgNorm): Pillow's 8-bit
 * Image.resize (src/libImaging/Resample.c: horizontal then vertical pass, 22-bit fixed-point coefficients, each pass rounded and
 * clipped to uint8), the centre crop, and torchvision's ToTensor + Normalize(0.5, 0.5), bit-exact.
 *   src [H0][W0][3] uint8 RGB (decoded image)            ->  out [3][H2][W2] fp32 in [-1, 1]
 *   x/ybounds [W1 | H1][2] = (first source index, taps <= kx | ky), x/ycoefs [kx | ky][W1 | H1] (tap-major) int32 with 22
 *   fractional bits: the tables of Resample.c precompute_coeffs + normalize_coeffs_8bpc for W0 -> W1 and H0 -> H1 (a dimension
 *   that does not change gets the identity table: bounds (i, 1), coefficient 1 << 22); the output is the window [crop_y0, crop_y0 + H2) x [crop_x0, crop_x0 + W2)
 *   of the resized image; [row0, row0 + rows) = the source rows those output rows read (union of their ybounds);
 *   lut [256] = the fp32 value of every byte after ImgNorm; tmp = workspace of rows * W2 * 3 bytes. */
int d3r_image_resize_crop_normalize(const uint8_t* src_dev, int32_t H0, int32_t W0, int32_t H1, int32_t W1,
                                    const int32_t* xbounds_dev, const int32_t* xcoefs_dev, int32_t kx,
                                    const int32_t* ybounds_dev, const int32_t* ycoefs_dev, int32_t ky, int32_t row0, int32_t rows,
                                    int32_t crop_x0, int32_t crop_y0, int32_t H2, int32_t W2, const float* lut_dev, uint8_t* tmp_dev,
                                    float* out_dev, void* stream);
/* The view stage of evaluation datasets (dust3r/datasets/base/base_stereo_view_dataset.py `_crop_resize_if_necessary` and
 * `__getitem__`) for n_views RGB-D frames of any mix of sizes in one call (three launches whatever the batch holds), bit-exact:
 *   image: the principal-point crop read in place, Pillow's 8-bit resize of it (as d3r_image_resize_crop_normalize), the final
 *   crop, ImgNorm -> img [3][H2][W2] fp32;
 *   depth: OpenCV's INTER_NEAREST resize of the same crop (source index min(floor(i * (1.0 / ((double)W1 / W0))), W0 - 1) per
 *   axis), the final crop -> depthmap [H2][W2] fp32; pts3d [H2][W2][3] fp32 = camera_pose applied (fp32, no fused multiply-add)
 *   to ((u - cu) * z / fu, (v - cv) * z / fv, z), the first two evaluated in fp64 and rounded once; valid [H2][W2] uint8 =
 *   z > 0 and the three coordinates finite.
 * With transpose != 0 (a portrait view) all four outputs are stored transposed: img [3][W2][H2], depthmap [W2][H2], pts3d
 * [W2][H2][3], valid [W2][H2].  The host plan (dust3r_b200/views.py) computes every field; the call validates the sizes and
 * windows of `desc` (host memory), uploads it to `desc_dev` (room for n_views descriptors, device memory, alive until the
 * kernels finish) with the `blocks` fields filled in, and launches.  lut [256] = the fp32 value of every byte after ImgNorm. */
typedef struct d3r_view_desc {
  const uint8_t* src;          /* RGB uint8, pixel (0, 0) of the principal-point crop; rows src_pitch pixels apart */
  const float* depth;          /* depth fp32, pixel (0, 0) of the principal-point crop; rows depth_pitch floats apart */
  int32_t src_pitch, depth_pitch;
  int32_t H0, W0;              /* principal-point crop = resize input */
  int32_t H1, W1;              /* resized size */
  int32_t crop_x0, crop_y0;    /* final crop window in the resized image */
  int32_t H2, W2;              /* output size before the landscape transpose */
  int32_t row0, rows;          /* crop rows the vertical pass reads: the union of the output rows' ybounds */
  int32_t transpose, reserved;
  const int32_t* xbounds;      /* [W1][2], xcoefs [kx][W1] tap-major: the Resample.c tables for W0 -> W1 */
  const int32_t* xcoefs;
  const int32_t* ybounds;      /* [H1][2], ycoefs [ky][H1] for H0 -> H1 */
  const int32_t* ycoefs;
  float fu, fv, cu, cv;        /* final camera intrinsics (before the transpose) */
  float pose[12];              /* camera-to-world rows [R | t], row-major; NaN when the frame has no pose */
  uint8_t* tmp;                /* workspace of rows * W2 * 3 bytes */
  float* img;
  float* depthmap;
  float* pts3d;
  uint8_t* valid;
  int64_t blocks[3];           /* first 256-thread block of this view in each launch; written by d3r_prepare_views */
} d3r_view_desc;

int32_t d3r_sizeof_view_desc(void);
int d3r_prepare_views(int32_t n_views, const d3r_view_desc* desc, d3r_view_desc* desc_dev, const float* lut_dev, void* stream);
/* Baseline JPEG decode (Pillow's np.asarray(exif_transpose(Image.open(f)).convert('RGB')), bit-exact): sequential Huffman,
 * 8-bit, 1 component or 3 YCbCr components at 4:4:4, 4:2:2 or 4:2:0, any restart interval.  The host parses the header into a
 * d3r_jpeg_desc; the compressed bytes [0, n_bytes) sit in device memory, the entropy-coded scan starts at scan_begin and ends at
 * the first marker other than RSTn.  out = uint8 [H][W][3] RGB after the EXIF orientation (W and H swapped for 5-8).
 * A stream that cannot be decoded exactly as libjpeg-turbo would sets bits of *status_dev (0 = decoded); the call itself only
 * fails on bad arguments.  Workspace: d3r_jpeg_decode_workspace_bytes(desc, n_bytes) bytes, no initialisation. */
typedef struct d3r_jpeg_huff {
  int32_t maxcode[18];     /* largest code of each length 1..16 (-1: none); [0] and [17] unused */
  int32_t valoff[18];      /* index into val of a code of each length, minus that code */
  uint16_t look[512];      /* next 9 bits -> (length << 8) | symbol, length 0 when the code is longer than 9 bits */
  uint8_t val[256];        /* symbols in code order, unused entries 0 */
} d3r_jpeg_huff;

typedef struct d3r_jpeg_desc {
  int32_t width, height;           /* frame size before the orientation */
  int32_t n_comp;                  /* 1 (grey) or 3 (YCbCr) */
  int32_t restart_interval;        /* MCUs per restart interval, 0 = none */
  int32_t orientation;             /* EXIF orientation 1..8 */
  int32_t reserved;
  int64_t scan_begin;              /* first byte of entropy-coded data, after the SOS header */
  int32_t h_samp[3], v_samp[3];    /* sampling factors, scan order */
  int32_t dc_table[3], ac_table[3];/* Huffman table slots 0..3 per component */
  uint16_t quant[3][64];           /* quantisation table per component, natural (row-major) order */
  d3r_jpeg_huff huff[8];           /* DC slots 0..3, then AC slots 0..3 */
} d3r_jpeg_desc;

#define D3R_JPEG_BAD_CODE 1        /* no Huffman code matches, or a run past coefficient 63 */
#define D3R_JPEG_SHORT 2           /* a restart interval or the scan ends before (or after) its last block, or not at EOI */
#define D3R_JPEG_BAD_RESTART 4     /* a restart marker out of sequence, or one without a restart interval */
#define D3R_JPEG_MARKER_COUNT 8    /* the scan ends before its last restart interval */
#define D3R_JPEG_RANGE 16          /* a DC value or an IDCT value outside the 16 / 32-bit lanes of Pillow's SIMD IDCT, or an IDCT
                                      output outside [-512, 511] (where Pillow saturates and libjpeg's C code wraps) */

int32_t d3r_sizeof_jpeg_desc(void);
int64_t d3r_jpeg_decode_workspace_bytes(const d3r_jpeg_desc* desc, int64_t n_bytes);
int d3r_jpeg_decode(const d3r_jpeg_desc* desc, const uint8_t* data_dev, int64_t n_bytes, uint8_t* out_dev, int32_t* status_dev,
                    void* workspace_dev, int64_t workspace_bytes, void* stream);

/* PNG decode (Pillow's np.asarray(exif_transpose(Image.open(f)).convert('RGB')), bit-exact): non-interlaced, 8-bit samples,
 * colour type 0 (grey), 2 (RGB), 3 (palette), 4 (grey + alpha) or 6 (RGBA).  The host walks the chunks into a d3r_png_desc and
 * concatenates every IDAT payload into one zlib stream of n_bytes (== desc->idat_bytes) bytes in device memory.  The stream is
 * inflated, its Adler-32 checked, the rows unfiltered and converted as convert('RGB') does (grey replicated, alpha dropped,
 * palette looked up, tRNS ignored).  out = uint8 [H][W][3] RGB after the EXIF orientation (W and H swapped for 5-8).
 * A stream the kernels cannot reproduce exactly as zlib + Pillow would sets bits of *status_dev (0 = decoded); the call itself
 * only fails on bad arguments.  Workspace: d3r_png_decode_workspace_bytes(desc, n_bytes) bytes, no initialisation. */
typedef struct d3r_png_desc {
  int32_t width, height;           /* image size before the orientation */
  int32_t color_type;              /* 0, 2, 3, 4 or 6 */
  int32_t orientation;             /* EXIF orientation 1..8 */
  int32_t palette_len;             /* PLTE entries (colour type 3: 1..256), 0 otherwise */
  int32_t reserved;
  int64_t idat_bytes;              /* bytes of the concatenated IDAT payloads (the zlib stream) */
  uint8_t palette[256][3];         /* PLTE, RGB; entries past palette_len unused */
} d3r_png_desc;

#define D3R_PNG_BAD_CODE 1         /* an invalid block header, code-length sequence, Huffman code or stored-block length */
#define D3R_PNG_FAR 2              /* a distance beyond the output produced so far */
#define D3R_PNG_SHORT 4            /* the stream ends early, data is left after the last block, the stream inflates to more or
                                      fewer bytes than the image rows, or it holds more blocks than the workspace records */
#define D3R_PNG_ADLER 8            /* Adler-32 mismatch */
#define D3R_PNG_FILTER 16          /* a row filter type above 4 */
#define D3R_PNG_PALETTE 32         /* a palette index at or past palette_len */

int32_t d3r_sizeof_png_desc(void);
int64_t d3r_png_decode_workspace_bytes(const d3r_png_desc* desc, int64_t n_bytes);
int d3r_png_decode(const d3r_png_desc* desc, const uint8_t* zdata_dev, int64_t n_bytes, uint8_t* out_dev, int32_t* status_dev,
                   void* workspace_dev, int64_t workspace_bytes, void* stream);

/* segment_sky (dust3r/viz.py:345-381, behind BasePCOptimizer.mask_sky, dust3r/cloud_opt/base_opt.py:289-295), bit-exact, for
 * n images of any mix of sizes in one call (seven launches whatever the content):
 *   rgb [total_px][3] uint8, image i = pixels [off[i], off[i] + hw[2i] * hw[2i+1]) row-major: the bytes uint8(255 * clip(img, 0, 1))
 *   -> sky_out [total_px] uint8 0 / 1.  OpenCV's 8-bit HSV of the bytes read as BGR, the reference's colour thresholds, a 5x5
 *   binary opening with zero padding, 8-connected components; a pixel is sky when its component has 2 * area > the largest
 *   component's area of its image (none when the opened mask is empty).
 * max_area = largest hw[2i] * hw[2i+1]; total_px = sum of the image areas (< 2^31); images must not overlap.  sky_out also serves
 * as scratch during the call.  The workspace (labels, areas, eroded mask, per-image maxima) needs
 * d3r_segment_sky_workspace_bytes(n_imgs, total_px) bytes (0 for an empty batch) and no initialisation. */
int64_t d3r_segment_sky_workspace_bytes(int32_t n_imgs, int64_t total_px);
int d3r_segment_sky(int32_t n_imgs, const int32_t* hw_dev, const int64_t* off_dev, int32_t max_area, int64_t total_px,
                    const uint8_t* rgb_dev, uint8_t* sky_out_dev, void* workspace_dev, int64_t workspace_bytes, void* stream);

/* Segmented lower nanmedian (torch.nanmedian(vals, dim=-1).values): vals [n_seg][seg_len] fp32 -> out [n_seg], element
 * (n - 1) / 2 of the sorted non-NaN values of each row, NaN for a row with none.  Radix select on order-preserving uint32 keys
 * (8-bit digits, most significant first): one memset and 4 x (histogram, select) launches whatever the content; -0 sorts below
 * +0.  n_seg <= 65535, seg_len < 2^32.  Workspace: d3r_nanmedian_workspace_bytes(n_seg) bytes, no initialisation. */
int64_t d3r_nanmedian_workspace_bytes(int32_t n_seg);
int d3r_segmented_nanmedian(int32_t n_seg, int64_t seg_len, const float* vals_dev, float* out_dev, void* workspace_dev,
                            int64_t workspace_bytes, void* stream);
/* The evaluation criteria of dust3r/losses.py (Regr3D, Regr3D_ShiftInv / _ScaleInv / _ScaleShiftInv with L21, ConfLoss) for B
 * pairs of views of n1 and n2 pixels, inference-only (no gradient):
 *   T [B][16] inv(camera_pose of view 1) row-major; gt1/gt2 [B][n][3] ground-truth points in world coordinates (anything at
 *   invalid pixels); valid1/valid2 [B][n] uint8 (nonzero = valid); pr1 / pr2 [B][n][3] predicted pts3d of view 1 and
 *   pts3d_in_other_view of view 2; conf1 / conf2 [B][n] (flag 16 only).
 *   flags: 1 'avg_dis' normalisation, 2 gt_scale, 4 shift-invariant (joint median depth), 8 scale-invariant (median centre and
 *   scale), 16 ConfLoss weighting with `alpha`, 32 dist_clip.  reduction: 0 mean, 1 sum, 2 none.
 *   out [7] fp32: the two views' distance (mean, 0 for an empty view | sum | with reduction 2 the mean, NaN for an empty view),
 *   the two views' confidence loss (mean, 0 for an empty view), the criterion's value (Regr3D: view 1 + view 2, ConfLoss: the two
 *   confidence losses; NaN with reduction 2), then the two valid counts as int32 bits.  With reduction 2, pix1 / pix2 (B * n
 *   floats each, or NULL) receive the distances of the valid pixels compacted in row-major (b, pixel) order and mask1 / mask2
 *   (B * n bytes each, or NULL) the valid mask.  fp64 sums reduced in a fixed order: two calls give the same bits.
 *   B * (n1 + n2) < 2^31, B <= 10922.  Workspace: d3r_criterion_workspace_bytes(B, n1, n2, flags) bytes, no initialisation. */
int64_t d3r_criterion_workspace_bytes(int32_t B, int64_t n1, int64_t n2, int32_t flags);
int d3r_criterion(int32_t B, int64_t n1, int64_t n2, int32_t flags, int32_t reduction, float dist_clip, float alpha,
                  const float* T_dev, const float* gt1_dev, const float* gt2_dev, const uint8_t* valid1_dev, const uint8_t* valid2_dev,
                  const float* pr1_dev, const float* pr2_dev, const float* conf1_dev, const float* conf2_dev, float* out_dev,
                  float* pix1_dev, float* pix2_dev, uint8_t* mask1_dev, uint8_t* mask2_dev, void* workspace_dev,
                  int64_t workspace_bytes, void* stream);


/* PnP-RANSAC (dust3r_visloc/localization.py run_pnp: cv2.solvePnPRansac with SOLVEPNP_SQPNP flags up to its final refinement)
 * on n >= 5 correspondences pts2d_dev fp32 [n][2] (pixels) / pts3d_dev fp32 [n][3] (world), pinhole fx, fy, cx, cy.
 * OpenCV's loop with 5-point EPnP hypotheses in fp64, its fp32 inlier test (squared reprojection error <= fp32(threshold^2))
 * and its stopping rule (confidence, at most max_iters hypotheses); the samples come from the counter-based generator of
 * csrc/pnp_core.h keyed by `seed`.  Device outputs: result_dev int32[4] = {best hypothesis (-1: none), its inlier count,
 * hypotheses evaluated, 1}; pose_dev fp64[12] = the best hypothesis' R (row-major, world -> camera) and t; mask_dev uint8[n]
 * its inliers.  workspace_dev: d3r_pnp_ransac_workspace_bytes(max_iters) bytes, 16-byte aligned. */
int64_t d3r_pnp_ransac_workspace_bytes(int32_t max_iters);
int d3r_pnp_ransac(int32_t n, const float* pts2d_dev, const float* pts3d_dev, double fx, double fy, double cx, double cy,
                   double threshold, double confidence, int32_t max_iters, int64_t seed, void* workspace_dev, int64_t workspace_bytes,
                   int32_t* result_dev, double* pose_dev, uint8_t* mask_dev, void* stream);
/* Hypotheses h0 .. h0 + n_hyp - 1 of d3r_pnp_ransac's sequence, without the loop: idx_dev int32[n_hyp][5] the samples (-1 when
 * none could be drawn), pose_dev fp64[n_hyp][12] the EPnP poses (0 when invalid), counts_dev int32[n_hyp] the inlier counts
 * (-1 when invalid). */
int d3r_pnp_hypotheses(int32_t n, const float* pts2d_dev, const float* pts3d_dev, double fx, double fy, double cx, double cy,
                       double threshold, int64_t seed, int32_t h0, int32_t n_hyp, int32_t* idx_dev, double* pose_dev,
                       int32_t* counts_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Path 1 — pairwise forward: replaces AsymmetricCroCo3DStereo.forward (dust3r/model.py:199-211 =
 * _encode_symmetrized :153-170, _decoder :172-191, downstream heads :193-208) as an encode call and a
 * decode call.  Weights are caller-owned device buffers, repacked once by the host side
 * (dust3r_b200/model.py: bf16 GEMM operands, fp32 biases / LayerNorm parameters).
 * ------------------------------------------------------------------------------------------ */
typedef struct d3r_linear { const void* w; const float* b; } d3r_linear;  /* w: bf16 [out][in]; b may be NULL */
typedef struct d3r_norm { const float* g; const float* b; } d3r_norm;     /* LayerNorm weight / bias (fp32)   */

typedef struct d3r_enc_block {      /* croco/models/blocks.py:114-130 */
  d3r_norm norm1, norm2;
  d3r_linear qkv, proj, fc1, fc2;
} d3r_enc_block;

typedef struct d3r_dec_block {      /* croco/models/blocks.py:171-191 */
  d3r_norm norm1, norm2, norm3, norm_y;
  d3r_linear qkv, proj;             /* self attention                                             */
  d3r_linear projq, projkv, cproj;  /* cross attention; projkv = rows of projk then projv          */
  d3r_linear fc1, fc2;
} d3r_dec_block;

typedef struct d3r_fusion {         /* FeatureFusionBlock_custom, croco/models/dpt_block.py:130-212 */
  d3r_linear rcu1_conv1, rcu1_conv2, rcu2_conv1, rcu2_conv2; /* 3x3, packed [Cout][9][Cin]           */
  d3r_linear out_conv;                                     /* 1x1 [256][256]                        */
} d3r_fusion;

typedef struct d3r_dpt_head {       /* DPTOutputAdapter_fix, dust3r/heads/dpt_head.py:20-65         */
  d3r_linear act_conv[4];           /* 1x1 convs on the 4 hooked token maps                        */
  d3r_linear act0_up;               /* ConvTranspose k4 s4 as GEMM  [(ky*4+kx)*96+co][ci]           */
  d3r_linear act1_up;               /* ConvTranspose k2 s2 as GEMM  [(ky*2+kx)*192+co][ci]          */
  d3r_linear act3_down;             /* 3x3 s2 p1 as GEMM over im2col [768][9*768]                   */
  d3r_linear layer_rn[4];           /* 3x3, no bias, packed                                        */
  d3r_fusion refine[4];             /* refinenet1..4                                               */
  d3r_linear head0;                 /* 3x3 256->128 packed                                         */
  d3r_linear head2;                 /* 3x3 128->128 packed                                         */
  const float* head4_w;             /* fp32 [nch][128]                                             */
  const float* head4_b;             /* fp32 [nch]                                                  */
} d3r_dpt_head;

typedef struct d3r_model {
  int32_t enc_dim, enc_depth, enc_heads, dec_dim, dec_depth, dec_heads, mlp_ratio, patch;
  int32_t head_type;                /* 0 = linear (LinearPts3d), 1 = dpt                            */
  int32_t nch;                      /* 3 + has_conf                                                */
  int32_t depth_mode;               /* 0 linear, 1 square, 2 exp  (postprocess.py:23-44)            */
  int32_t conf_mode;                /* 0 none, 1 exp, 2 sigmoid   (postprocess.py:47-58)            */
  float conf_min, conf_max, ln_eps;
  int32_t hooks[4];                 /* DPT hooks into [enc_out, dec_1..dec_L] (dpt_head.py:110)     */
  int32_t rope_max_pos;
  const float* rope_cos;            /* [rope_max_pos][16]                                          */
  const float* rope_sin;
  d3r_linear patch_embed;           /* [enc_dim][3*patch*patch]                                    */
  const d3r_enc_block* enc;         /* host array [enc_depth]                                      */
  d3r_norm enc_norm;
  d3r_linear decoder_embed;
  const d3r_dec_block* dec1;        /* dec_blocks   (host array [dec_depth])                       */
  const d3r_dec_block* dec2;        /* dec_blocks2                                                 */
  d3r_norm dec_norm;
  const d3r_dpt_head* dpt[2];       /* downstream_head1/2 when head_type == 1                      */
  d3r_linear lin_head[2];           /* downstream_head{1,2}.proj when head_type == 0               */
} d3r_model;

/* sizeof(d3r_model) as compiled into the library (binding self-check). */
int d3r_sizeof_model(void);

/* The forward is two calls on one stream.
 * d3r_encode_images: imgs (n,3,H,W) fp32 in [-1,1] -> feat (n, H/16, W/16, enc_dim) bf16, caller-owned: the
 * encoder's output after enc_norm (model.py:128-140), the tensor the decoder and DPT hook 0 read.  A symmetrised batch
 * (model.py:153-170) encodes only its even half; two views of different sizes (model.py:147-151) are encoded by one
 * call each.
 * d3r_decode_pairs: decoders + heads for B pairs; pair b is (image idx1[b] of feat1, image idx2[b] of feat2),
 * idx HOST int32[B], indices in [0, n1) / [0, n2).  feat1 and feat2 may be the same buffer when the sizes are equal.
 * Features must be 16-byte aligned.  Outputs (fp32, device): pts3d_1 (B,H1,W1,3), conf_1 (B,H1,W1) in view1's frame
 * for view1; pts3d_2 (B,H2,W2,3) / conf_2 (B,H2,W2) for view2 ('pts3d_in_other_view').  conf pointers may be NULL
 * when the model has no confidence channel.
 * Each image's features, and each pair's outputs, are independent of the rest of their call, so features can be kept
 * between calls (each image of a multi-view scene encoded once, however many pairs it appears in).  Debug taps 1-4
 * apply to the encode call, 5 and up to the decode call. */
int64_t d3r_encode_workspace_bytes(const d3r_model* m, int32_t n, int32_t H, int32_t W);
int d3r_encode_images(const d3r_model* m, const float* imgs_dev, int32_t n, int32_t H, int32_t W, void* feat_dev,
                      void* workspace_dev, int64_t workspace_bytes, void* stream);
int64_t d3r_decode_workspace_bytes(const d3r_model* m, int32_t B, int32_t H1, int32_t W1, int32_t H2, int32_t W2);
int d3r_decode_pairs(const d3r_model* m, const void* feat1_dev, int32_t n1, int32_t H1, int32_t W1, const void* feat2_dev,
                     int32_t n2, int32_t H2, int32_t W2, const int32_t* idx1_host, const int32_t* idx2_host, int32_t B,
                     float* pts3d_1, float* conf_1, float* pts3d_2, float* conf_2, void* workspace_dev,
                     int64_t workspace_bytes, void* stream);

/* Optional taps for the parity tests: when non-NULL, fp32 copies of intermediate stages are written.
 * (set with d3r_forward_set_debug before a call; cleared after it).  stage ids in DESIGN.md. */
int d3r_forward_set_debug(int32_t stage_id, float* out_dev, int64_t capacity_floats);

#ifdef __cplusplus
}
#endif
#endif /* DUST3R_B200_H_ */
