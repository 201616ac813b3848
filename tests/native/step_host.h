// Host side of the step decoders (JPEG, PNG): runs a codec's `decode` launch sequence with g++, calling the per-thread body
// Codec::step<S> of csrc/<codec>_core.h for every thread index a launch would cover, plus the ragged tail of its last
// 128-thread block.  Pointers are HOST pointers.  step_host_main is the stand-alone program a harness becomes for the
// AddressSanitizer runs of the tests.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

template <class Codec>
struct HostLauncher {
  using Plan = typename Codec::Plan;
  using Work = typename Codec::Work;
  std::function<void(int S, const Plan&, const Work&)> after_step;   // optional: called after every launch
  void zero(void* p, long long bytes) { std::memset(p, 0, (size_t)bytes); }
  void copy_desc(void* dst, const typename Codec::Desc* src) { std::memcpy(dst, src, sizeof(typename Codec::Desc)); }
  template <int S>
  void launch(long long n, int k, const Plan& P, Work& w) {
    const long long threads = (n + 127) / 128 * 128;
    for (long long t = 0; t < threads; ++t) Codec::template step<S>(t, k, P, w);
    if (after_step) after_step(S, P, w);
  }
};

template <class Codec>
long long host_workspace_bytes(const typename Codec::Desc* desc, long long n_bytes) {
  typename Codec::Plan P;
  if (Codec::make_plan(*desc, n_bytes, P)) return 0;
  return typename Codec::Layout(P).bytes;
}

// Decodes `data` into `out` (out_h x out_w x 3) and `status`, leaving the plan and the workspace pointers in P and w for the
// caller to inspect; false on a rejected descriptor.
template <class Codec>
bool host_decode(const typename Codec::Desc* desc, const uint8_t* data, long long n_bytes, uint8_t* out, int32_t* status,
                 void* workspace, typename Codec::Plan& P, typename Codec::Work& w, HostLauncher<Codec> l = {}) {
  if (Codec::make_plan(*desc, n_bytes, P)) return false;
  const typename Codec::Layout lay(P);
  char* ws = static_cast<char*>(workspace);
  w = lay.work(ws);
  w.*Codec::kInput = data;
  w.out = out;
  w.status = status;
  Codec::decode(l, P, lay, w, *desc, ws);
  return true;
}

inline std::vector<uint8_t> slurp(const char* path) {
  std::vector<uint8_t> v;
  FILE* f = std::fopen(path, "rb");
  if (!f) std::exit(2);
  int c;
  while ((c = std::fgetc(f)) != EOF) v.push_back((uint8_t)c);
  std::fclose(f);
  return v;
}

// argv = pairs of (descriptor file, input file); every buffer is allocated at its exact size, so a read past the input is
// reported.  fit (optional) adapts a descriptor to the input's length.  Prints one status word per pair.
template <class Codec>
int step_host_main(int argc, char** argv, void (*fit)(typename Codec::Desc&, long long) = nullptr) {
  using Desc = typename Codec::Desc;
  for (int i = 1; i + 1 < argc; i += 2) {
    const std::vector<uint8_t> d = slurp(argv[i]);
    if (d.size() != sizeof(Desc)) return 3;
    Desc* desc = (Desc*)std::malloc(sizeof(Desc));
    std::memcpy(desc, d.data(), sizeof(Desc));
    const std::vector<uint8_t> file = slurp(argv[i + 1]);
    if (fit) fit(*desc, (long long)file.size());
    uint8_t* data = (uint8_t*)std::malloc(file.size());
    std::memcpy(data, file.data(), file.size());
    const long long ws_bytes = host_workspace_bytes<Codec>(desc, (long long)file.size());
    typename Codec::Plan P;
    if (!ws_bytes || Codec::make_plan(*desc, (long long)file.size(), P)) return 4;
    void* ws = std::malloc((size_t)ws_bytes);
    uint8_t* out = (uint8_t*)std::malloc((size_t)P.W * P.H * 3);
    int32_t status = 0;
    typename Codec::Work w;
    if (!host_decode<Codec>(desc, data, (long long)file.size(), out, &status, ws, P, w)) return 5;
    std::printf("%d\n", status);
    std::free(out);
    std::free(ws);
    std::free(data);
    std::free(desc);
  }
  return 0;
}
