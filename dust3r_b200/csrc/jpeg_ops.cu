// Baseline JPEG decode on the GPU, bit-identical to Pillow (libjpeg-turbo): the per-thread bodies and the launch sequence are in
// jpeg_core.h (shared with the host harness tests/native/jpeg_host.cpp), the kernels and the entry-point body in
// step_decode.cuh.  Every step is one thread per item (subsequence, group, DC slice, 8x8 block, pixel).
#include "jpeg_core.h"
#include "step_decode.cuh"

using namespace d3r;

extern "C" int32_t d3r_sizeof_jpeg_desc(void) { return (int32_t)sizeof(d3r_jpeg_desc); }

extern "C" int64_t d3r_jpeg_decode_workspace_bytes(const d3r_jpeg_desc* desc, int64_t n_bytes) {
  return step_decode_workspace_bytes<jpeg::Codec>(desc, n_bytes);
}

extern "C" int d3r_jpeg_decode(const d3r_jpeg_desc* desc, const uint8_t* data_dev, int64_t n_bytes, uint8_t* out_dev,
                               int32_t* status_dev, void* workspace_dev, int64_t workspace_bytes, void* stream) {
  D3R_CHECK_ARG(n_bytes > 0, "d3r_jpeg_decode: n_bytes = %lld", (long long)n_bytes);
  return step_decode<jpeg::Codec>(desc, data_dev, n_bytes, out_dev, status_dev, workspace_dev, workspace_bytes, stream);
}
