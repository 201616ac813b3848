// Attention entry points: kernel selection and the C ABI (the kernel lives in attention_wgmma.cu).
//   O[b, i, h*64 + d] = softmax_j(scale * q[b,i,h,:] . k[b,j,h,:]) v[b,j,h,d]      head dim 64 (all DUSt3R heads), bf16 in/out
// replaces the materialised (B,H,N,N) fp32 attention matrix of croco/models/blocks.py:105-109 / :161-165.
#include "d3r_common.cuh"
#include "elementwise.h"

namespace d3r {
namespace attn {

// 3 (default): P V with P in registers; 2: the same dataflow with P through shared memory, kept as the A/B reference --
// both produce the same bits.
static int g_impl = 3;

void set_impl(int impl) { g_impl = (impl == 2) ? 2 : 3; }

int attention_hd64(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* out,
                   long long ldo, int B, int heads, int Nq, int Nk, float scale, cudaStream_t st) {
  return attention_hd64_wgmma(q, ldq, k, ldk, v, ldv, out, ldo, B, heads, Nq, Nk, scale, g_impl == 2, st);
}

}  // namespace attn
}  // namespace d3r

extern "C" void d3r_set_attention_impl(int32_t impl) { d3r::attn::set_impl(impl); }

extern "C" int d3r_attention_hd64(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out,
                                  int64_t ldo, int32_t B, int32_t heads, int32_t Nq, int32_t Nk, float scale, void* stream) {
  return d3r::attn::attention_hd64(q, ldq, k, ldk, v, ldv, out, ldo, B, heads, Nq, Nk, scale, (cudaStream_t)stream);
}
