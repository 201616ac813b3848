// Host harness of the PNG decoder: compiles dust3r_b200/csrc/png_core.h -- the very per-thread bodies and launch sequence the
// CUDA kernels of csrc/png_ops.cu run -- with g++ and runs them through step_host.h.  tests/test_png_host.py compares the
// result with Pillow bit for bit and builds it a second time under -fsanitize=address to show that corrupt streams are reported
// without reading outside the buffers.  Same argument list as d3r_png_decode minus the stream; pointers are HOST pointers here.
#include "../../dust3r_b200/csrc/png_core.h"
#include "step_host.h"

using namespace d3r::png;

extern "C" long long png_host_workspace_bytes(const d3r_png_desc* desc, long long n_bytes) {
  return host_workspace_bytes<Codec>(desc, n_bytes);
}

// 0 on success, -1 on a rejected descriptor.  blocks (optional, capacity max_blocks) receives the start bit of every block of
// the chain, n_blocks their number; speculative (optional) the number of them the chain took from a speculative record.
extern "C" int png_host_decode(const d3r_png_desc* desc, const uint8_t* data, long long n_bytes, uint8_t* out, int32_t* status,
                               void* workspace, long long* blocks, long long max_blocks, long long* n_blocks,
                               long long* speculative) {
  Plan P;
  Work w;
  if (!host_decode<Codec>(desc, data, n_bytes, out, status, workspace, P, w)) return -1;
  const long long nb = (long long)w.ctl[0];
  if (n_blocks) *n_blocks = nb;
  long long spec = 0;
  for (long long i = 0; i < nb; ++i) {
    if (blocks && i < max_blocks) blocks[i] = w.chain[i].start;
    const long long p = w.chain[i].start, s = p / (8ll * kSubBytes);
    for (int j = 0; j < w.nrec[s]; ++j)
      if (w.rec[s * kSlots + j].start == p && w.rec[s * kSlots + j].err == 0) {
        ++spec;
        break;
      }
  }
  if (speculative) *speculative = spec;
  return 0;
}

#ifdef PNG_HOST_MAIN
// the stream file's length is the descriptor's IDAT length
int main(int argc, char** argv) {
  return step_host_main<Codec>(argc, argv, [](d3r_png_desc& d, long long n) { d.idat_bytes = n; });
}
#endif
