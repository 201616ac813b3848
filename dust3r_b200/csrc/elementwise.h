// Internal host API of the bandwidth-bound glue kernels (elementwise.cu) and attention (attention_wgmma.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstddef>

namespace d3r {
namespace ew {
int layernorm(const float* x, const float* g, const float* b, void* out_bf16, const int* row_map, int M, int C, float eps, cudaStream_t st);
int cast_f32_bf16(const float* x, void* out, size_t n, cudaStream_t st);
int gather_images_bf16(const void* in, void* out, const int* img_map_dev, int n_out_imgs, int rows_per_img, int C, cudaStream_t st);
int patch_im2col16(const float* img, void* out, int B, int H, int W, cudaStream_t st);
int upsample2x_bf16(const void* x, void* out, int B, int H, int W, int C, int Ho, int Wo, cudaStream_t st);
int im2col_3x3_s2_bf16(const void* x, void* out, int B, int H, int W, int C, cudaStream_t st);
int linear_head_postprocess(const float* feat, float* pts3d, float* conf, int B, int gh, int gw, int nch, int depth_mode,
                            int conf_mode, float cmin, float cmax, cudaStream_t st);
}  // namespace ew
namespace attn {
// O[b, i, h*64 + d] = softmax_j(scale * q[b,i,h,:] . k[b,j,h,:]) v[b,j,h,d];  head dim 64, bf16 in/out.
// q rows: (b*Nq + i)*ldq + h*64 ; k/v rows: (b*Nk + j)*ldk(v) + h*64.
int attention_hd64(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* out,
                   long long ldo, int B, int heads, int Nq, int Nk, float scale, cudaStream_t st);
}  // namespace attn
}  // namespace d3r
