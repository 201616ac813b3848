// Host harness of the PNG decoder: compiles dust3r_b200/csrc/png_core.h -- the very per-thread bodies and launch sequence the
// CUDA kernels of csrc/png_ops.cu run -- with g++ and runs every step for every thread index a launch would cover (plus the
// ragged tail of its last block).  tests/test_png_host.py compares the result with Pillow bit for bit and builds it a second time
// under -fsanitize=address to show that corrupt streams are reported without reading outside the buffers.  Same argument list as
// d3r_png_decode minus the stream; pointers are HOST pointers here.
#include <cstring>
#include <vector>

#include "../../dust3r_b200/csrc/png_core.h"

using namespace d3r::png;

namespace {

struct HostLauncher {
  void zero(void* p, long long bytes) { std::memset(p, 0, (size_t)bytes); }
  void copy_desc(void* dst, const d3r_png_desc* src) { std::memcpy(dst, src, sizeof(d3r_png_desc)); }
  template <int S>
  void launch(long long n, int k, const Plan& P, Work& w) {
    const long long threads = (n + 127) / 128 * 128;
    for (long long t = 0; t < threads; ++t) step<S>(t, k, P, w);
  }
};

}  // namespace

extern "C" long long png_host_workspace_bytes(const d3r_png_desc* desc, long long n_bytes) {
  Plan P;
  if (make_plan(*desc, n_bytes, P)) return 0;
  return Layout(P).bytes;
}

// 0 on success, -1 on a rejected descriptor.  blocks (optional, capacity max_blocks) receives the start bit of every block of
// the chain, n_blocks their number; speculative (optional) the number of them the chain took from a speculative record.
extern "C" int png_host_decode(const d3r_png_desc* desc, const uint8_t* data, long long n_bytes, uint8_t* out, int32_t* status,
                               void* workspace, long long* blocks, long long max_blocks, long long* n_blocks,
                               long long* speculative) {
  Plan P;
  if (make_plan(*desc, n_bytes, P)) return -1;
  const Layout lay(P);
  char* ws = static_cast<char*>(workspace);
  Work w = lay.work(ws);
  w.z = data;
  w.out = out;
  w.status = status;
  HostLauncher l;
  decode(l, P, lay, w, *desc, ws);
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
// Stand-alone form for the AddressSanitizer run: argv = pairs of (descriptor file, zlib stream file); every buffer is allocated
// at its exact size, so a read past the stream is reported.  Prints one status word per pair.
#include <cstdio>
#include <cstdlib>

static std::vector<uint8_t> slurp(const char* path) {
  std::vector<uint8_t> v;
  FILE* f = std::fopen(path, "rb");
  if (!f) std::exit(2);
  int c;
  while ((c = std::fgetc(f)) != EOF) v.push_back((uint8_t)c);
  std::fclose(f);
  return v;
}

int main(int argc, char** argv) {
  for (int i = 1; i + 1 < argc; i += 2) {
    const std::vector<uint8_t> d = slurp(argv[i]);
    if (d.size() != sizeof(d3r_png_desc)) return 3;
    d3r_png_desc* desc = (d3r_png_desc*)std::malloc(sizeof(d3r_png_desc));
    std::memcpy(desc, d.data(), sizeof(d3r_png_desc));
    const std::vector<uint8_t> file = slurp(argv[i + 1]);
    desc->idat_bytes = (long long)file.size();
    uint8_t* data = (uint8_t*)std::malloc(file.size());
    std::memcpy(data, file.data(), file.size());
    const long long ws_bytes = png_host_workspace_bytes(desc, (long long)file.size());
    Plan P;
    if (!ws_bytes || make_plan(*desc, (long long)file.size(), P)) return 4;
    void* ws = std::malloc((size_t)ws_bytes);
    uint8_t* out = (uint8_t*)std::malloc((size_t)P.W * P.H * 3);
    int32_t status = 0;
    if (png_host_decode(desc, data, (long long)file.size(), out, &status, ws, nullptr, 0, nullptr, nullptr)) return 5;
    std::printf("%d\n", status);
    std::free(out);
    std::free(ws);
    std::free(data);
    std::free(desc);
  }
  return 0;
}
#endif
