// Host harness of the JPEG decoder: compiles dust3r_b200/csrc/jpeg_core.h -- the very per-thread bodies and launch sequence the
// CUDA kernels of csrc/jpeg_ops.cu run -- with g++ and runs every step for every thread index a launch would cover (plus the
// ragged tail of its last block).  tests/test_jpeg_host.py compares the result with Pillow bit for bit and builds it a second time
// under -fsanitize=address to show that corrupt streams are reported without reading outside the buffers.  Same argument list as
// d3r_jpeg_decode minus the stream; pointers are HOST pointers here.
#include <cstring>
#include <vector>

#include "../../dust3r_b200/csrc/jpeg_core.h"

using namespace d3r::jpeg;

namespace {

struct HostLauncher {
  std::vector<Cursor>* phase1_end = nullptr;   // when set: a copy of the phase-1 end states
  void zero(void* p, long long bytes) { std::memset(p, 0, (size_t)bytes); }
  void copy_desc(void* dst, const d3r_jpeg_desc* src) { std::memcpy(dst, src, sizeof(d3r_jpeg_desc)); }
  template <int S>
  void launch(long long n, int k, const Plan& P, Work& w) {
    const long long threads = (n + 127) / 128 * 128;
    for (long long t = 0; t < threads; ++t) step<S>(t, k, P, w);
    if (S == kPhase1 && phase1_end) phase1_end->assign(w.end, w.end + P.nsub);
  }
};

}  // namespace

extern "C" long long jpeg_host_workspace_bytes(const d3r_jpeg_desc* desc, long long n_bytes) {
  Plan P;
  if (make_plan(*desc, n_bytes, P)) return 0;
  return Layout(P).bytes;
}

// 0 on success, -1 on a rejected descriptor; subsequences / sync_rounds (optional) report the parallel decode's shape
extern "C" int jpeg_host_decode(const d3r_jpeg_desc* desc, const uint8_t* data, long long n_bytes, uint8_t* out, int32_t* status,
                                void* workspace, long long* subsequences, int* sync_rounds) {
  Plan P;
  if (make_plan(*desc, n_bytes, P)) return -1;
  const Layout lay(P);
  char* ws = static_cast<char*>(workspace);
  Work w = lay.work(ws);
  w.data = data;
  w.out = out;
  w.status = status;
  HostLauncher l;
  decode(l, P, lay, w, *desc, ws);
  if (subsequences) *subsequences = P.nsub;
  if (sync_rounds) {
    int k = 0;
    while (k < kSyncRounds && w.changed[k] > 0) ++k;
    *sync_rounds = w.ctl[1] ? kSyncRounds + 1 : k;       // kSyncRounds + 1: the sequential finish had work to do
  }
  return 0;
}

// The speculative decode against a sequential one: every subsequence's synchronised start state must be the state a single
// decoder from the start of the scan holds at the first symbol boundary at or after that subsequence's first byte.  Returns the
// number of subsequences that differ (0), or -1 on a rejected descriptor.  resynced (optional) = subsequences whose phase-1
// guess was wrong.
extern "C" long long jpeg_host_check_sync(const d3r_jpeg_desc* desc, const uint8_t* data, long long n_bytes, void* workspace,
                                          long long* resynced) {
  Plan P;
  if (make_plan(*desc, n_bytes, P)) return -1;
  const Layout lay(P);
  char* ws = static_cast<char*>(workspace);
  Work w = lay.work(ws);
  std::vector<uint8_t> out((size_t)P.out_w * P.out_h * 3);
  int32_t status = 0;
  w.data = data;
  w.out = out.data();
  w.status = &status;
  std::vector<Cursor> p1;
  HostLauncher l;
  l.phase1_end = &p1;
  decode(l, P, lay, w, *desc, ws);
  long long bad = 0, wrong = 0;
  Cursor c{P.scan_begin * 8, 0, 0, 0, 0};
  for (long long s = 0; s < P.nsub; ++s) {
    if (!same(c, w.start[s])) ++bad;
    if (s + 1 < P.nsub) {
      if (!same(p1[s], w.end[s])) ++wrong;
      run(P, *w.desc, data, c, sub_end_bit(P, scan_end(P, w), s), nullptr);   // one sequential decoder, stopped at every boundary
    }
  }
  if (resynced) *resynced = wrong;
  return bad;
}

#ifdef JPEG_HOST_MAIN
// Stand-alone form for the AddressSanitizer run: argv = pairs of (descriptor file, JPEG file); every buffer is allocated at its
// exact size, so a read past the compressed bytes is reported.  Prints one status word per pair.
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
    if (d.size() != sizeof(d3r_jpeg_desc)) return 3;
    d3r_jpeg_desc* desc = (d3r_jpeg_desc*)std::malloc(sizeof(d3r_jpeg_desc));
    std::memcpy(desc, d.data(), sizeof(d3r_jpeg_desc));
    const std::vector<uint8_t> file = slurp(argv[i + 1]);
    uint8_t* data = (uint8_t*)std::malloc(file.size());
    std::memcpy(data, file.data(), file.size());
    const long long ws_bytes = jpeg_host_workspace_bytes(desc, (long long)file.size());
    Plan P;
    if (!ws_bytes || make_plan(*desc, (long long)file.size(), P)) return 4;
    void* ws = std::malloc((size_t)ws_bytes);
    uint8_t* out = (uint8_t*)std::malloc((size_t)P.W * P.H * 3);
    int32_t status = 0;
    if (jpeg_host_decode(desc, data, (long long)file.size(), out, &status, ws, nullptr, nullptr)) return 5;
    std::printf("%d\n", status);
    std::free(out);
    std::free(ws);
    std::free(data);
    std::free(desc);
  }
  return 0;
}
#endif
