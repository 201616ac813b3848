// Per-thread bodies and launch sequence of the baseline JPEG decoder (csrc/jpeg_ops.cu), written once for device AND host: the
// CUDA kernels call step<S>(t, ...) with t = blockIdx.x * blockDim.x + threadIdx.x, tests/native/jpeg_host.cpp compiles this very
// header with g++ and calls the same bodies in a loop over t, through the same `decode` sequence, so the bit-exactness against
// Pillow (libjpeg-turbo) and the bounds of every read are checked on machines without a GPU.
//
// What is restated (libjpeg-turbo as Pillow drives it: JDCT_ISLOW, do_fancy_upsampling, JCS_RGB output):
//   entropy decoding   jdhuff.c decode_mcu for baseline sequential Huffman scans, restart markers resetting the DC predictions
//   dequantisation     coefficient * quantiser, then jidctint.c jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2, DESCALE rounding,
//                      the 10-bit wrap-around range limit of IDCT_range_limit)
//   upsampling         jdsample.c h2v1_fancy_upsample / h2v2_fancy_upsample (triangle filter, alternating +1 / +2 and +8 / +7
//                      biases, edge columns and replicated edge rows), the box upsamplers when the chroma width is <= 2
//   colour             jdcolor.c ycc_rgb_convert with its 16-bit fixed-point tables; grey replicated to RGB as convert('RGB')
//   orientation        ImageOps.exif_transpose as an index map on the store
//
// Parallel entropy decoding (Weissenberger & Schmidt, "Massively parallel Huffman decoding on GPUs", ICPP 2018): the scan is cut
// into subsequences of kSubBytes raw bytes, up to the first marker other than RSTn (found first, so that whatever follows EOI --
// MPF previews, gain maps, vendor trailers -- is never decoded).  Phase 1 decodes every subsequence from a guessed state (first
// byte, block 0 of the MCU, coefficient 0) up to its end.  A state is (bit position, block in MCU, coefficient index).  Up to
// kSyncRounds parallel rounds then give every subsequence the end state of its predecessor and decode it again where that start
// changed; each round carries a corrected state one subsequence further, and most photographs are consistent after a handful of
// rounds.  Whatever is still inconsistent after them (streams without end-of-block codes, such as noise at quality 100, can
// stay out of step for their whole length) is finished by one thread that walks from the first inconsistent subsequence,
// decoding only where its state differs from the stored start and skipping ahead through stored end states where it agrees:
// the decode always completes, in the worst case as one sequential decoder.  A prefix over the per-subsequence (restart markers passed, blocks decoded)
// gives each subsequence its first block, a second pass writes the coefficients, and per-component prefix sums that reset at
// every restart marker turn DC differences into DC values.  Byte stuffing (FF 00) and markers are resolved by the bit reader
// itself; every read is bounded by the byte count the host passed.  A stream the decoder cannot complete the way libjpeg would
// sets bits of the status word instead (the caller then decodes that file with Pillow).
#pragma once
#include <stdint.h>

#include "../../include/dust3r_b200.h"

#include "hd.h"

namespace d3r {
namespace jpeg {

constexpr int kSubBytes = 256;          // raw bytes per subsequence
constexpr int kSyncRounds = 8;          // parallel sync rounds before the sequential finish
constexpr int kMarkerScanBytes = 32;    // bytes per thread of the end-of-scan search
constexpr int kMaxUnits = 6;            // blocks per MCU: 4:2:0 = 4 Y + Cb + Cr
constexpr int kDcSliceMcus = 64;        // MCUs per thread of the DC prefix sums
constexpr long long kDone = 0x7fffffffffffffffll;   // bit position of a cursor that reached the end of the scan

// status word bits
constexpr int kBadCode = D3R_JPEG_BAD_CODE, kShort = D3R_JPEG_SHORT, kBadRestart = D3R_JPEG_BAD_RESTART,
              kMarkerCount = D3R_JPEG_MARKER_COUNT, kRange = D3R_JPEG_RANGE;

#if !defined(__CUDACC__)
struct int2 { int x, y; };
struct int4 { int x, y, z, w; };
#endif

// jutils.c jpeg_natural_order: zig-zag index -> row-major index
#define D3R_JPEG_NATURAL {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, \
                          41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, \
                          30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63}
#if defined(__CUDACC__)
__constant__ unsigned char kNaturalDev[64] = D3R_JPEG_NATURAL;
#endif
static const unsigned char kNaturalHost[64] = D3R_JPEG_NATURAL;

D3R_HD int natural(int k) {
#if defined(__CUDA_ARCH__)
  return kNaturalDev[k];
#else
  return kNaturalHost[k];
#endif
}

// Everything the kernels need besides the tables, derived once from the descriptor on the host (make_plan)
struct Plan {
  int W, H, ncomp, hmax, vmax, orientation;
  int h[3], v[3], dc[3], ac[3];
  int mcux, mcuy, bpm;                      // MCUs per row / column, blocks per MCU
  int unit_comp[kMaxUnits], unit_dy[kMaxUnits], unit_dx[kMaxUnits];
  int restart;                              // MCUs per restart interval, 0 = none
  long long mcus, blocks, seg_blocks;       // total MCUs, total blocks, blocks per restart interval (all blocks without restarts)
  long long nseg;                           // restart intervals
  long long scan_begin, n_bytes;            // scan = bytes [scan_begin, n_bytes) of the buffer
  long long nsub, ngrp, grp, ndc;           // subsequences, groups of `grp` subsequences, DC slices
  long long plane_off[3];                   // component sample planes in the workspace
  int plane_w[3], dw[3], dh[3];             // plane pitch, downsampled width / height
  int out_w, out_h;                         // after the orientation
};

// A decoding position and what was seen on the way.  Compared states use pos / unit / zz only.
struct Cursor {
  long long pos;            // raw bit position of the next unread bit (byte * 8 + bit), kDone at the end of the scan
  int unit, zz;             // block in the MCU, next coefficient (0 = DC)
  int markers, blocks;      // restart markers passed, blocks completed since the last one (or the start)
};

struct Work {                // workspace pointers
  const d3r_jpeg_desc* desc;
  Cursor* start;            // [nsub] start state of every subsequence
  Cursor* end;              // [nsub] end state decoding from start
  int* dirty;               // [nsub]
  int* changed;             // [kSyncRounds + 1]
  unsigned long long* ctl;  // [2]: n_bytes - first end-of-scan marker, nsub - first subsequence inconsistent after the rounds
  int2* grp;                // [ngrp] (markers, blocks) of each group of subsequences
  int2* first;              // [nsub] (restart interval, block in it) at the start of every subsequence
  int16_t* coef;            // [blocks][64] natural order
  int* dcdiff;              // [blocks]
  int4* dcsum;              // [ndc] (reset seen, DC sums per component) of each slice
  uint8_t* planes;
  const uint8_t* data;      // compressed bytes
  uint8_t* out;             // [out_h][out_w][3]
  int* status;
};

D3R_HD void flag(int* status, int bit) {
#if defined(__CUDA_ARCH__)
  atomicOr(status, bit);
#else
  *status |= bit;
#endif
}

D3R_HD bool same(const Cursor& a, const Cursor& b) { return a.pos == b.pos && a.unit == b.unit && a.zz == b.zz; }

// ------------------------------------------------------------------------------------------------ bit reader
// Up to 8 data bytes from raw byte p, MSB first; returns the number of data bits and leaves in *stop the raw position where it
// stopped (a marker, or the end of the buffer) when fewer than 64 bits were found.  FF 00 is a data byte FF.
D3R_HD int gather(const uint8_t* d, long long n, long long p, uint64_t& w, long long& stop) {
  w = 0;
  int nb = 0;
  while (nb < 64) {
    if (p >= n) break;
    const uint8_t b = d[p];
    if (b == 0xFF) {
      if (p + 1 < n && d[p + 1] == 0) p += 2;
      else break;
    } else {
      p += 1;
    }
    w |= (uint64_t)b << (56 - nb);
    nb += 8;
  }
  stop = p;
  return nb;
}

// raw position after `k` data bytes starting at the data byte p (all of them inside what gather just read)
D3R_HD long long skip_data(const uint8_t* d, long long p, int k) {
  for (int i = 0; i < k; ++i) p += d[p] == 0xFF ? 2 : 1;
  return p;
}

// Coefficient sink of the write pass; the decode-only passes run with none.
struct Sink {
  const Plan* P;
  Work* w;
  long long seg, inseg;     // restart interval and its block index at the start of the run
};

// blocks of restart interval s
D3R_HD long long seg_len(const Plan& P, long long s) {
  return s < P.nseg - 1 ? P.seg_blocks : P.blocks - (P.nseg - 1) * P.seg_blocks;
}

D3R_HD long long sink_block(const Sink& k, const Cursor& c, long long& seg) {
  seg = k.seg + c.markers;
  const long long inseg = (c.markers == 0 ? k.inseg : 0) + c.blocks;
  if (seg >= k.P->nseg || inseg >= seg_len(*k.P, seg)) return -1;
  return seg * k.P->seg_blocks + inseg;
}

// Decodes from c until its position reaches end_bit (or the scan ends).  Sync passes: sink == nullptr.
D3R_HD void run(const Plan& P, const d3r_jpeg_desc& D, const uint8_t* d, Cursor& c, long long end_bit, Sink* sink) {
  const long long n = P.n_bytes;
  while (c.pos < end_bit) {
    const long long p = c.pos >> 3;
    const int off = (int)(c.pos & 7);
    uint64_t w;
    long long stop;
    const int nb = gather(d, n, p, w, stop);
    const int avail = nb - off;
    bool incomplete = avail <= 0;
    int len = 0, sym = 0;
    const uint64_t bits = incomplete ? 0 : w << off;
    if (!incomplete) {
      const int comp = P.unit_comp[c.unit];
      const d3r_jpeg_huff& T = D.huff[c.zz == 0 ? P.dc[comp] : 4 + P.ac[comp]];
      const unsigned e = T.look[bits >> 55];
      len = e >> 8;
      sym = e & 255;
      if (len == 0) {
        len = 10;
        long long code = (long long)(bits >> 54);
        while (len <= 16 && code > T.maxcode[len]) code = (long long)(bits >> (64 - ++len));
        if (len > 16) {
          if (avail < 16) {
            incomplete = true;
          } else {             // no such code: mark, skip to the end of this subsequence (a guessed start, or a corrupt stream)
            if (sink) flag(sink->w->status, kBadCode);
            c.pos = end_bit;
            c.unit = 0;
            c.zz = 0;
            break;
          }
        } else {
          sym = T.val[(unsigned)(T.valoff[len] + (int)code) & 255u];
        }
      }
    }
    const int s = c.zz == 0 ? sym : (sym & 15);
    if (!incomplete && len + s > avail) incomplete = true;
    if (incomplete) {
      // the data before the marker (padding bits after the last block of an interval) holds no further symbol: the marker
      // ends the interval
      const bool rst = stop + 1 < n && d[stop] == 0xFF && d[stop + 1] >= 0xD0 && d[stop + 1] <= 0xD7;
      if (sink) {
        long long seg;
        const long long inseg = (c.markers == 0 ? sink->inseg : 0) + c.blocks;
        seg = sink->seg + c.markers;
        if (seg >= P.nseg || inseg != seg_len(P, seg)) flag(sink->w->status, kShort);
        if (rst ? (P.restart == 0 || seg + 1 >= P.nseg || (d[stop + 1] & 7) != (seg & 7)) : seg != P.nseg - 1)
          flag(sink->w->status, rst ? kBadRestart : kMarkerCount);
        // the scan must end at EOI: Pillow refuses a file whose data run out first
        if (!rst && !(stop + 1 < n && d[stop] == 0xFF && d[stop + 1] == 0xD9)) flag(sink->w->status, kShort);
      }
      if (rst) {
        c.pos = (stop + 2) * 8;
        c.unit = 0;
        c.zz = 0;
        c.markers += 1;
        c.blocks = 0;
        continue;
      }
      c.pos = kDone;            // every cursor that reached the end compares equal, whatever block it was in
      c.unit = 0;
      c.zz = 0;
      break;
    }
    int v = 0;
    if (s) {
      v = (int)((bits << len) >> (64 - s));
      if (v < (1 << (s - 1))) v += (int)(~0u << s) + 1;
    }
    int k = c.zz;
    bool block_done;
    if (k == 0) {
      if (sink) {
        long long seg;
        const long long b = sink_block(*sink, c, seg);
        if (b >= 0) sink->w->dcdiff[b] = v;
      }
      k = 1;
      block_done = false;
    } else {
      const int r = sym >> 4;
      if (s) {
        k += r;
        if (k > 63) {          // libjpeg would store it in coefficient 63: never produced by an encoder, decoded by Pillow
          if (sink) flag(sink->w->status, kBadCode);
          k = 63;
        } else if (sink) {
          long long seg;
          const long long b = sink_block(*sink, c, seg);
          if (b >= 0) sink->w->coef[b * 64 + natural(k)] = (int16_t)v;
        }
        k += 1;
        block_done = k >= 64;
      } else if (r == 15) {
        k += 16;
        if (k > 64 && sink) flag(sink->w->status, kBadCode);
        block_done = k >= 64;
      } else {
        block_done = true;
      }
    }
    const int adv = off + len + s;
    c.pos = skip_data(d, p, adv >> 3) * 8 + (adv & 7);
    if (block_done) {
      c.zz = 0;
      c.unit = c.unit + 1 == P.bpm ? 0 : c.unit + 1;
      c.blocks += 1;
    } else {
      c.zz = k;
    }
  }
}

// raw position of the first marker other than RSTn after the scan start (n_bytes when there is none)
D3R_HD long long scan_end(const Plan& P, const Work& w) { return P.n_bytes - (long long)w.ctl[0]; }

// the last subsequence before the scan end runs until the scan ends, so that the end marker is always checked
D3R_HD long long sub_end_bit(const Plan& P, long long se, long long s) {
  const long long e = P.scan_begin + (s + 1) * kSubBytes;
  return e < se ? e * 8 : kDone;
}

D3R_HD void atomic_max(unsigned long long* p, unsigned long long v) {
#if defined(__CUDA_ARCH__)
  atomicMax(p, v);
#else
  if (v > *p) *p = v;
#endif
}

// ------------------------------------------------------------------------------------------------ per-thread bodies
enum Step { kScanEnd, kPhase1, kUpdate, kRedecode, kFinish, kGroupSum, kGroupScan, kWrite, kDcSum, kDcScan, kIdct, kColour };

// thread t = bytes [scan_begin + 32 t, + 32): the first FF there that is not stuffing (FF 00) and not RSTn ends the scan.  The
// second byte of FF 00 or FF Dn is never FF, so every FF the bit reader would stop at is a candidate here, and the earliest one
// is where it stops.
D3R_HD void scan_end_body(long long t, const Plan& P, Work& w) {
  const long long n = P.n_bytes;
  const long long b = P.scan_begin + t * kMarkerScanBytes;
  if (b >= n) return;
  const long long e = b + kMarkerScanBytes < n ? b + kMarkerScanBytes : n;
  for (long long p = b; p < e; ++p) {
    if (w.data[p] != 0xFF) continue;
    if (p + 1 < n) {
      const uint8_t m = w.data[p + 1];
      if (m == 0 || (m >= 0xD0 && m <= 0xD7)) continue;
    }
    atomic_max(w.ctl, (unsigned long long)(n - p));
    return;
  }
}

// phase 1: subsequence t from a guessed state (its first data byte, block 0, coefficient 0); subsequence 0 starts exactly there.
// Subsequences past the end of the scan are finished before they start.
D3R_HD void phase1_body(long long t, const Plan& P, Work& w) {
  if (t >= P.nsub) return;
  const long long se = scan_end(P, w);
  long long b = P.scan_begin + t * kSubBytes;
  if (t > 0 && b >= se) {
    w.start[t] = w.end[t] = Cursor{kDone, 0, 0, 0, 0};
    return;
  }
  if (t > 0 && w.data[b - 1] == 0xFF) b += 1;         // second byte of a stuffed FF 00 or of a marker
  Cursor c{b * 8, 0, 0, 0, 0};
  w.start[t] = c;
  run(P, *w.desc, w.data, c, sub_end_bit(P, se, t), nullptr);
  w.end[t] = c;
}

// sync round k: subsequence t takes its predecessor's end state; round kSyncRounds only records the first subsequence whose
// start still disagrees, for the sequential finish
D3R_HD void update_body(long long t, int k, const Plan& P, Work& w) {
  if (t >= P.nsub || t == 0) return;
  if (k > 0 && w.changed[k - 1] == 0) return;
  Cursor want = w.end[t - 1];
  if (same(want, w.start[t])) return;
  if (k == kSyncRounds) {
    atomic_max(w.ctl + 1, (unsigned long long)(P.nsub - t));
    return;
  }
  want.markers = 0;
  want.blocks = 0;
  w.start[t] = want;
  w.dirty[t] = 1;
#if defined(__CUDA_ARCH__)
  atomicAdd(w.changed + k, 1);
#else
  w.changed[k] += 1;
#endif
}

D3R_HD void redecode_body(long long t, const Plan& P, Work& w) {
  if (t >= P.nsub || !w.dirty[t]) return;
  w.dirty[t] = 0;
  Cursor c = w.start[t];
  run(P, *w.desc, w.data, c, sub_end_bit(P, scan_end(P, w), t), nullptr);
  w.end[t] = c;
}

// one thread (t == 0): from the first inconsistent subsequence on, a sequential decoder that re-decodes a subsequence only where
// its state differs from the stored start, and otherwise takes the stored end state (decoded from that very start)
D3R_HD void finish_body(long long t, const Plan& P, Work& w) {
  if (t != 0 || w.ctl[1] == 0) return;
  const long long se = scan_end(P, w);
  long long j = P.nsub - (long long)w.ctl[1];
  Cursor cur = w.end[j - 1];
  for (; j < P.nsub; ++j) {
    if (same(cur, w.start[j])) {
      cur = w.end[j];
      continue;
    }
    cur.markers = 0;
    cur.blocks = 0;
    w.start[j] = cur;
    run(P, *w.desc, w.data, cur, sub_end_bit(P, se, j), nullptr);
    w.end[j] = cur;
  }
}

// (markers, blocks) of a then b
D3R_HD int2 combine(int2 a, int2 b) {
  int2 r;
  r.x = a.x + b.x;
  r.y = b.x > 0 ? b.y : a.y + b.y;
  return r;
}

D3R_HD void group_sum_body(long long t, const Plan& P, Work& w) {
  if (t >= P.ngrp) return;
  int2 acc{0, 0};
  const long long e = (t + 1) * P.grp < P.nsub ? (t + 1) * P.grp : P.nsub;
  for (long long s = t * P.grp; s < e; ++s) acc = combine(acc, int2{w.end[s].markers, w.end[s].blocks});
  w.grp[t] = acc;
}

// the prefix of the groups before t is folded by every thread (a few hundred broadcast loads), then t's own subsequences
D3R_HD void group_scan_body(long long t, const Plan& P, Work& w) {
  if (t >= P.ngrp) return;
  int2 acc{0, 0};
  for (long long g = 0; g < t; ++g) acc = combine(acc, w.grp[g]);
  const long long e = (t + 1) * P.grp < P.nsub ? (t + 1) * P.grp : P.nsub;
  for (long long s = t * P.grp; s < e; ++s) {
    w.first[s] = acc;
    acc = combine(acc, int2{w.end[s].markers, w.end[s].blocks});
  }
}

D3R_HD void write_body(long long t, const Plan& P, Work& w) {
  if (t >= P.nsub) return;
  Cursor c = w.start[t];
  if (c.pos == kDone) return;
  c.markers = 0;
  c.blocks = 0;
  Sink k{&P, &w, w.first[t].x, w.first[t].y};
  run(P, *w.desc, w.data, c, sub_end_bit(P, scan_end(P, w), t), &k);
}

// DC: per-slice sums after the last restart in the slice, per component
D3R_HD void dc_sum_body(long long t, const Plan& P, Work& w) {
  if (t >= P.ndc) return;
  int4 acc{0, 0, 0, 0};
  const long long m1 = (t + 1) * kDcSliceMcus < P.mcus ? (t + 1) * kDcSliceMcus : P.mcus;
  for (long long m = t * kDcSliceMcus; m < m1; ++m) {
    if (P.restart > 0 && m % P.restart == 0) acc = int4{1, 0, 0, 0};
    for (int u = 0; u < P.bpm; ++u) {
      const int d = w.dcdiff[m * P.bpm + u];
      const int c = P.unit_comp[u];
      if (c == 0) acc.y += d;
      else if (c == 1) acc.z += d;
      else acc.w += d;
    }
  }
  w.dcsum[t] = acc;
}

D3R_HD void dc_scan_body(long long t, const Plan& P, Work& w) {
  if (t >= P.ndc) return;
  long long pred[3] = {0, 0, 0};       // 64-bit: a crafted stream may push a running DC sum far outside 32 bits
  for (long long g = 0; g < t; ++g) {
    const int4 s = w.dcsum[g];
    if (s.x) pred[0] = pred[1] = pred[2] = 0;
    pred[0] += s.y;
    pred[1] += s.z;
    pred[2] += s.w;
  }
  const long long m1 = (t + 1) * kDcSliceMcus < P.mcus ? (t + 1) * kDcSliceMcus : P.mcus;
  for (long long m = t * kDcSliceMcus; m < m1; ++m) {
    if (P.restart > 0 && m % P.restart == 0) pred[0] = pred[1] = pred[2] = 0;
    for (int u = 0; u < P.bpm; ++u) {
      const long long b = m * P.bpm + u;
      long long& p = pred[P.unit_comp[u]];
      p += w.dcdiff[b];
      if (p < -32768 || p > 32767) flag(w.status, kRange);
      w.coef[b * 64] = (int16_t)p;
    }
  }
}

// jidctint.c constants (CONST_BITS 13)
constexpr long long F0_298 = 2446, F0_390 = 3196, F0_541 = 4433, F0_765 = 6270, F0_899 = 7373, F1_175 = 9633, F1_501 = 12299,
                    F1_847 = 15137, F1_961 = 16069, F2_053 = 16819, F2_562 = 20995, F3_072 = 25172;

D3R_HD long long descale(long long x, int n) { return (x + (1ll << (n - 1))) >> n; }

D3R_HD bool fits16(long long v) { return v >= -32768 && v <= 32767; }
D3R_HD bool fits32(long long v) { return v >= -2147483648ll && v <= 2147483647ll; }

// One 8-point pass of jpeg_idct_islow: in[0..7], results descaled by `sh`.  Returns false where the SIMD IDCT Pillow runs
// (libjpeg-turbo's jidctint-avx2 / -sse2) could differ from this C arithmetic: it forms the pairwise input sums in 16 bits
// (paddw / psubw, wrapping) and the products and output sums in 32 bits (pmaddwd / paddd, wrapping), so any such value outside
// those widths is reported instead of restated.
D3R_HD bool idct8(const long long* in, long long* out, int sh) {
  bool ok = fits16(in[0] + in[4]) && fits16(in[0] - in[4]) && fits16(in[2] + in[6]) && fits16(in[7] + in[1]) &&
            fits16(in[5] + in[3]) && fits16(in[7] + in[3]) && fits16(in[5] + in[1]) &&
            fits16(in[7] + in[3] + in[5] + in[1]);
  long long z2 = in[2], z3 = in[6];
  long long z1 = (z2 + z3) * F0_541;
  long long tmp2 = z1 + z3 * (-F1_847);
  long long tmp3 = z1 + z2 * F0_765;
  long long tmp0 = (in[0] + in[4]) * 8192;
  long long tmp1 = (in[0] - in[4]) * 8192;
  const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = in[7];
  tmp1 = in[5];
  tmp2 = in[3];
  tmp3 = in[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * F1_175;
  tmp0 *= F0_298;
  tmp1 *= F2_053;
  tmp2 *= F3_072;
  tmp3 *= F1_501;
  z1 *= -F0_899;
  z2 *= -F2_562;
  z3 *= -F1_961;
  z4 *= -F0_390;
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  const long long round = 1ll << (sh - 1);
  ok = ok && fits32(tmp10 + tmp3 + round) && fits32(tmp10 - tmp3 + round) && fits32(tmp11 + tmp2 + round) &&
       fits32(tmp11 - tmp2 + round) && fits32(tmp12 + tmp1 + round) && fits32(tmp12 - tmp1 + round) &&
       fits32(tmp13 + tmp0 + round) && fits32(tmp13 - tmp0 + round) && fits32(tmp0) && fits32(tmp1) && fits32(tmp2) &&
       fits32(tmp3) && fits32(tmp10) && fits32(tmp11) && fits32(tmp12) && fits32(tmp13);
  out[0] = descale(tmp10 + tmp3, sh);
  out[7] = descale(tmp10 - tmp3, sh);
  out[1] = descale(tmp11 + tmp2, sh);
  out[6] = descale(tmp11 - tmp2, sh);
  out[2] = descale(tmp12 + tmp1, sh);
  out[5] = descale(tmp12 - tmp1, sh);
  out[3] = descale(tmp13 + tmp0, sh);
  out[4] = descale(tmp13 - tmp0, sh);
  return ok;
}

// IDCT_range_limit: the low 10 bits as a signed value, plus 128, clamped
D3R_HD uint8_t range_limit(long long x) {
  int v = (int)(x & 1023);
  if (v >= 512) v -= 1024;
  v += 128;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// thread t = block t of the scan (MCU-major): dequantise, IDCT, store the 8x8 samples into its component plane
D3R_HD void idct_body(long long t, const Plan& P, Work& w) {
  if (t >= P.blocks) return;
  const long long mcu = t / P.bpm;
  const int u = (int)(t - mcu * P.bpm);
  const int c = P.unit_comp[u];
  const long long by = (mcu / P.mcux) * P.v[c] + P.unit_dy[u], bx = (mcu % P.mcux) * P.h[c] + P.unit_dx[u];
  const int16_t* in = w.coef + t * 64;
  const uint16_t* q = w.desc->quant[c];
  long long ws[64], col[8], res[8];
  bool range_ok = true;
  for (int x = 0; x < 8; ++x) {
    for (int y = 0; y < 8; ++y) {
      col[y] = (long long)in[8 * y + x] * q[8 * y + x];
      range_ok = range_ok && fits16(col[y]);          // the SIMD code dequantises with a 16-bit multiply (pmullw)
    }
    range_ok = idct8(col, res, 13 - 2) && range_ok;
    for (int y = 0; y < 8; ++y) {
      ws[8 * y + x] = res[y];
      range_ok = range_ok && fits16(res[y]);          // pass-1 results are packed to 16 bits (packssdw, saturating)
    }
  }
  uint8_t* dst = w.planes + P.plane_off[c] + by * 8 * P.plane_w[c] + bx * 8;
  for (int y = 0; y < 8; ++y) {
    range_ok = idct8(ws + 8 * y, res, 13 + 2 + 3) && range_ok;
    for (int x = 0; x < 8; ++x) {
      // the C range limit wraps the low 10 bits, the SIMD store saturates (packsswb): equal only inside [-512, 511]
      range_ok = range_ok && res[x] >= -512 && res[x] <= 511;
      dst[(long long)y * P.plane_w[c] + x] = range_limit(res[x]);
    }
  }
  if (!range_ok) flag(w.status, kRange);
}

// chroma sample at full resolution (x, y) of component c: libjpeg-turbo's fancy upsampling, box upsampling for narrow planes
D3R_HD int upsample(const Plan& P, const uint8_t* pl, int c, int x, int y) {
  const int pw = P.plane_w[c], dw = P.dw[c], dh = P.dh[c];
  const bool h2 = P.h[c] * 2 == P.hmax, v2 = P.v[c] * 2 == P.vmax;
  if (!h2) return pl[(long long)y * pw + x];                 // 4:4:4
  const int i = x >> 1;
  if (dw <= 2) return pl[(long long)(v2 ? y >> 1 : y) * pw + i];
  if (!v2) {                                                  // h2v1
    const uint8_t* r = pl + (long long)y * pw;
    if ((x & 1) == 0) return i == 0 ? r[0] : (r[i] * 3 + r[i - 1] + 1) >> 2;
    return i == dw - 1 ? r[i] : (r[i] * 3 + r[i + 1] + 2) >> 2;
  }
  const int row = y >> 1;                                     // h2v2
  int nrow = (y & 1) ? row + 1 : row - 1;
  nrow = nrow < 0 ? 0 : (nrow > dh - 1 ? dh - 1 : nrow);
  const uint8_t* r0 = pl + (long long)row * pw;
  const uint8_t* r1 = pl + (long long)nrow * pw;
  const int cs = r0[i] * 3 + r1[i];
  if ((x & 1) == 0) {
    if (i == 0) return (cs * 4 + 8) >> 4;
    return (cs * 3 + r0[i - 1] * 3 + r1[i - 1] + 8) >> 4;
  }
  if (i == dw - 1) return (cs * 4 + 7) >> 4;
  return (cs * 3 + r0[i + 1] * 3 + r1[i + 1] + 7) >> 4;
}

D3R_HD uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// thread t = source pixel (x, y): upsample, ycc_rgb_convert, store at its place after exif_transpose
D3R_HD void colour_body(long long t, const Plan& P, Work& w) {
  if (t >= (long long)P.W * P.H) return;
  const int y = (int)(t / P.W), x = (int)(t - (long long)y * P.W);
  const int Y = w.planes[P.plane_off[0] + (long long)y * P.plane_w[0] + x];
  int R = Y, G = Y, B = Y;
  if (P.ncomp == 3) {
    const int cb = upsample(P, w.planes + P.plane_off[1], 1, x, y) - 128;
    const int cr = upsample(P, w.planes + P.plane_off[2], 2, x, y) - 128;
    R = clamp255(Y + ((91881 * cr + 32768) >> 16));
    G = clamp255(Y + ((-22554 * cb + 32768 + -46802 * cr) >> 16));
    B = clamp255(Y + ((116130 * cb + 32768) >> 16));
  }
  int ox = x, oy = y;
  const int W = P.W, H = P.H;
  switch (P.orientation) {
    case 2: ox = W - 1 - x; break;                              // FLIP_LEFT_RIGHT
    case 3: ox = W - 1 - x; oy = H - 1 - y; break;              // ROTATE_180
    case 4: oy = H - 1 - y; break;                              // FLIP_TOP_BOTTOM
    case 5: ox = y; oy = x; break;                              // TRANSPOSE
    case 6: ox = H - 1 - y; oy = x; break;                      // ROTATE_270
    case 7: ox = H - 1 - y; oy = W - 1 - x; break;              // TRANSVERSE
    case 8: ox = y; oy = W - 1 - x; break;                      // ROTATE_90
    default: break;
  }
  uint8_t* o = w.out + ((long long)oy * P.out_w + ox) * 3;
  o[0] = (uint8_t)R;
  o[1] = (uint8_t)G;
  o[2] = (uint8_t)B;
}

template <int S>
D3R_HD void step(long long t, int k, const Plan& P, Work& w) {
  if (S == kScanEnd) scan_end_body(t, P, w);
  else if (S == kPhase1) phase1_body(t, P, w);
  else if (S == kUpdate) update_body(t, k, P, w);
  else if (S == kRedecode) redecode_body(t, P, w);
  else if (S == kFinish) finish_body(t, P, w);
  else if (S == kGroupSum) group_sum_body(t, P, w);
  else if (S == kGroupScan) group_scan_body(t, P, w);
  else if (S == kWrite) write_body(t, P, w);
  else if (S == kDcSum) dc_sum_body(t, P, w);
  else if (S == kDcScan) dc_scan_body(t, P, w);
  else if (S == kIdct) idct_body(t, P, w);
  else colour_body(t, P, w);
}

// ------------------------------------------------------------------------------------------------ host side
inline long long align_up(long long b) { return (b + 255) / 256 * 256; }

// Plan of a descriptor, or an error message (argument checks before any launch)
inline const char* make_plan(const d3r_jpeg_desc& D, long long n_bytes, Plan& P) {
  P = Plan{};
  if (D.width < 1 || D.height < 1 || D.width > 65535 || D.height > 65535) return "image size outside [1, 65535]";
  if (D.n_comp != 1 && D.n_comp != 3) return "only 1 or 3 components";
  if (D.orientation < 1 || D.orientation > 8) return "orientation outside [1, 8]";
  if (D.restart_interval < 0) return "negative restart interval";
  if (D.scan_begin < 2 || D.scan_begin >= n_bytes) return "scan start outside the buffer";
  P.W = D.width;
  P.H = D.height;
  P.ncomp = D.n_comp;
  P.orientation = D.orientation;
  P.restart = D.restart_interval;
  P.hmax = P.vmax = 1;
  for (int c = 0; c < P.ncomp; ++c) {
    if (D.dc_table[c] < 0 || D.dc_table[c] > 3 || D.ac_table[c] < 0 || D.ac_table[c] > 3) return "Huffman table index outside [0, 3]";
    P.h[c] = D.h_samp[c];
    P.v[c] = D.v_samp[c];
    P.dc[c] = D.dc_table[c];
    P.ac[c] = D.ac_table[c];
    P.hmax = P.h[c] > P.hmax ? P.h[c] : P.hmax;
    P.vmax = P.v[c] > P.vmax ? P.v[c] : P.vmax;
  }
  if (P.ncomp == 1) {
    if (P.h[0] != 1 || P.v[0] != 1) return "grey images must have sampling 1x1";
  } else {
    const bool chroma11 = P.h[1] == 1 && P.v[1] == 1 && P.h[2] == 1 && P.v[2] == 1;
    const bool luma = (P.h[0] == 1 && P.v[0] == 1) || (P.h[0] == 2 && P.v[0] == 1) || (P.h[0] == 2 && P.v[0] == 2);
    if (!chroma11 || !luma) return "sampling must be 4:4:4, 4:2:2 or 4:2:0";
  }
  for (int i = 0; i < 8; ++i)
    for (int j = 0; j < 512; ++j)
      if ((D.huff[i].look[j] >> 8) > 9) return "Huffman lookahead entry longer than 9 bits";
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 256; ++j)
      if (D.huff[i].val[j] > 15) return "DC Huffman symbol above 15";
  P.mcux = (P.W + 8 * P.hmax - 1) / (8 * P.hmax);
  P.mcuy = (P.H + 8 * P.vmax - 1) / (8 * P.vmax);
  P.bpm = 0;
  for (int c = 0; c < P.ncomp; ++c)
    for (int dy = 0; dy < P.v[c]; ++dy)
      for (int dx = 0; dx < P.h[c]; ++dx) {
        P.unit_comp[P.bpm] = c;
        P.unit_dy[P.bpm] = dy;
        P.unit_dx[P.bpm] = dx;
        ++P.bpm;
      }
  P.mcus = (long long)P.mcux * P.mcuy;
  P.blocks = P.mcus * P.bpm;
  P.nseg = P.restart > 0 ? (P.mcus + P.restart - 1) / P.restart : 1;
  P.seg_blocks = P.restart > 0 ? (long long)P.restart * P.bpm : P.blocks;
  P.scan_begin = D.scan_begin;
  P.n_bytes = n_bytes;
  P.nsub = (n_bytes - D.scan_begin + kSubBytes - 1) / kSubBytes;
  P.grp = P.nsub / 1024 + 1;
  P.ngrp = (P.nsub + P.grp - 1) / P.grp;
  P.ndc = (P.mcus + kDcSliceMcus - 1) / kDcSliceMcus;
  long long off = 0;
  for (int c = 0; c < P.ncomp; ++c) {
    P.plane_w[c] = P.mcux * P.h[c] * 8;
    P.plane_off[c] = off;
    off += align_up((long long)P.plane_w[c] * P.mcuy * P.v[c] * 8);
    P.dw[c] = (int)(((long long)P.W * P.h[c] + P.hmax - 1) / P.hmax);
    P.dh[c] = (int)(((long long)P.H * P.v[c] + P.vmax - 1) / P.vmax);
  }
  const bool swap = P.orientation >= 5;
  P.out_w = swap ? P.H : P.W;
  P.out_h = swap ? P.W : P.H;
  return nullptr;
}

// workspace: [desc][start][end][dirty][changed][grp][first][dcsum][dcdiff][coef][planes], each 256-byte aligned
struct Layout {
  long long desc, start, end, dirty, changed, ctl, grp, first, dcsum, dcdiff, coef, planes, bytes;
  explicit Layout(const Plan& P) {
    desc = 0;
    start = desc + align_up(sizeof(d3r_jpeg_desc));
    end = start + align_up(P.nsub * (long long)sizeof(Cursor));
    dirty = end + align_up(P.nsub * (long long)sizeof(Cursor));
    changed = dirty + align_up(4 * P.nsub);
    ctl = changed + align_up(4 * (kSyncRounds + 1));
    grp = ctl + align_up(16);
    first = grp + align_up(8 * P.ngrp);
    dcsum = first + align_up(8 * P.nsub);
    dcdiff = dcsum + align_up(16 * P.ndc);
    coef = dcdiff + align_up(4 * P.blocks);
    planes = coef + align_up(128 * P.blocks);
    long long pl = 0;
    for (int c = 0; c < P.ncomp; ++c) pl += align_up((long long)P.plane_w[c] * P.mcuy * P.v[c] * 8);
    bytes = planes + pl;
  }
  Work work(char* ws) const {
    Work w{};
    w.desc = reinterpret_cast<const d3r_jpeg_desc*>(ws + desc);
    w.start = reinterpret_cast<Cursor*>(ws + start);
    w.end = reinterpret_cast<Cursor*>(ws + end);
    w.dirty = reinterpret_cast<int*>(ws + dirty);
    w.changed = reinterpret_cast<int*>(ws + changed);
    w.ctl = reinterpret_cast<unsigned long long*>(ws + ctl);
    w.grp = reinterpret_cast<int2*>(ws + grp);
    w.first = reinterpret_cast<int2*>(ws + first);
    w.dcsum = reinterpret_cast<int4*>(ws + dcsum);
    w.dcdiff = reinterpret_cast<int*>(ws + dcdiff);
    w.coef = reinterpret_cast<int16_t*>(ws + coef);
    w.planes = reinterpret_cast<uint8_t*>(ws + planes);
    return w;
  }
};

// The launch sequence, shared by the CUDA entry point and the host harness.  L provides
//   zero(ptr, bytes), copy_desc(dst, src), and template <int S> launch(n_threads, k, plan, work).
template <class L>
void decode(L& l, const Plan& P, const Layout& lay, Work& w, const d3r_jpeg_desc& desc, char* ws) {
  l.copy_desc(ws + lay.desc, &desc);
  l.zero(w.status, 4);
  l.zero(ws + lay.dirty, lay.grp - lay.dirty);                        // dirty flags, round counters, scan end, first inconsistency
  l.template launch<kScanEnd>((P.n_bytes - P.scan_begin + kMarkerScanBytes - 1) / kMarkerScanBytes, 0, P, w);
  l.zero(ws + lay.dcdiff, lay.planes - lay.dcdiff);                   // DC differences, coefficients
  l.template launch<kPhase1>(P.nsub, 0, P, w);
  for (int k = 0; k < kSyncRounds; ++k) {
    l.template launch<kUpdate>(P.nsub, k, P, w);
    l.template launch<kRedecode>(P.nsub, k, P, w);
  }
  l.template launch<kUpdate>(P.nsub, kSyncRounds, P, w);
  l.template launch<kFinish>(1, 0, P, w);
  l.template launch<kGroupSum>(P.ngrp, 0, P, w);
  l.template launch<kGroupScan>(P.ngrp, 0, P, w);
  l.template launch<kWrite>(P.nsub, 0, P, w);
  l.template launch<kDcSum>(P.ndc, 0, P, w);
  l.template launch<kDcScan>(P.ndc, 0, P, w);
  l.template launch<kIdct>(P.blocks, 0, P, w);
  l.template launch<kColour>((long long)P.W * P.H, 0, P, w);
}

// What the step-decoder launchers (csrc/step_decode.cuh, tests/native/step_host.h) need of this codec
struct Codec {
  using Desc = d3r_jpeg_desc;
  using Plan = jpeg::Plan;
  using Work = jpeg::Work;
  using Layout = jpeg::Layout;
  static constexpr const char* kEntry = "d3r_jpeg_decode";
  static constexpr const char* kTag = "jpeg_decode";
  static constexpr const uint8_t* Work::*kInput = &Work::data;
  static const char* make_plan(const Desc& D, long long n_bytes, Plan& P) { return jpeg::make_plan(D, n_bytes, P); }
  template <class L>
  static void decode(L& l, const Plan& P, const Layout& lay, Work& w, const Desc& desc, char* ws) {
    jpeg::decode(l, P, lay, w, desc, ws);
  }
  template <int S>
  D3R_HD static void step(long long t, int k, const Plan& P, Work& w) { jpeg::step<S>(t, k, P, w); }
  // compulsory traffic: the compressed bytes (read about three times), coefficients out and in, planes out and in, RGB out
  static double traffic(const Plan& P, long long n_bytes) {
    return 3.0 * double(n_bytes) + 2.0 * 132.0 * double(P.blocks) + 3.0 * double(P.W) * P.H * (P.ncomp == 3 ? 2 : 1);
  }
  static int launches(const Plan&) { return 2 * kSyncRounds + 12; }
};

}  // namespace jpeg
}  // namespace d3r
