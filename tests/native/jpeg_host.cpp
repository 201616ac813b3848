// Host harness of the JPEG decoder: compiles dust3r_b200/csrc/jpeg_core.h -- the very per-thread bodies and launch sequence the
// CUDA kernels of csrc/jpeg_ops.cu run -- with g++ and runs them through step_host.h.  tests/test_jpeg_host.py compares the
// result with Pillow bit for bit and builds it a second time under -fsanitize=address to show that corrupt streams are reported
// without reading outside the buffers.  Same argument list as d3r_jpeg_decode minus the stream; pointers are HOST pointers here.
#include <vector>

#include "../../dust3r_b200/csrc/jpeg_core.h"
#include "step_host.h"

using namespace d3r::jpeg;

extern "C" long long jpeg_host_workspace_bytes(const d3r_jpeg_desc* desc, long long n_bytes) {
  return host_workspace_bytes<Codec>(desc, n_bytes);
}

// 0 on success, -1 on a rejected descriptor; subsequences / sync_rounds (optional) report the parallel decode's shape
extern "C" int jpeg_host_decode(const d3r_jpeg_desc* desc, const uint8_t* data, long long n_bytes, uint8_t* out, int32_t* status,
                                void* workspace, long long* subsequences, int* sync_rounds) {
  Plan P;
  Work w;
  if (!host_decode<Codec>(desc, data, n_bytes, out, status, workspace, P, w)) return -1;
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
  std::vector<uint8_t> out((size_t)P.out_w * P.out_h * 3);
  int32_t status = 0;
  std::vector<Cursor> p1;   // the phase-1 end states
  HostLauncher<Codec> l;
  l.after_step = [&](int S, const Plan& plan, const Work& work) {
    if (S == kPhase1) p1.assign(work.end, work.end + plan.nsub);
  };
  Work w;
  host_decode<Codec>(desc, data, n_bytes, out.data(), &status, workspace, P, w, l);
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
int main(int argc, char** argv) { return step_host_main<Codec>(argc, argv); }
#endif
