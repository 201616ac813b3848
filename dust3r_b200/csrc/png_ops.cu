// PNG decode on the GPU, bit-identical to Pillow: the per-thread bodies and the launch sequence are in png_core.h (shared with
// the host harness tests/native/png_host.cpp), the kernels and the entry-point body in step_decode.cuh.  Every step is one
// thread per item (stream byte, subsequence, block, inflated byte, Adler segment, row).
#include "png_core.h"
#include "step_decode.cuh"

using namespace d3r;

extern "C" int32_t d3r_sizeof_png_desc(void) { return (int32_t)sizeof(d3r_png_desc); }

extern "C" int64_t d3r_png_decode_workspace_bytes(const d3r_png_desc* desc, int64_t n_bytes) {
  return step_decode_workspace_bytes<png::Codec>(desc, n_bytes);
}

extern "C" int d3r_png_decode(const d3r_png_desc* desc, const uint8_t* zdata_dev, int64_t n_bytes, uint8_t* out_dev,
                              int32_t* status_dev, void* workspace_dev, int64_t workspace_bytes, void* stream) {
  return step_decode<png::Codec>(desc, zdata_dev, n_bytes, out_dev, status_dev, workspace_dev, workspace_bytes, stream);
}
