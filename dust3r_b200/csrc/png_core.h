// Per-thread bodies and launch sequence of the PNG decoder (csrc/png_ops.cu), written once for device AND host: the CUDA kernels
// call step<S>(t, ...) with t = blockIdx.x * blockDim.x + threadIdx.x, tests/native/png_host.cpp compiles this very header with
// g++ and calls the same bodies in a loop over t, through the same `decode` sequence, so the bit-exactness against Pillow and
// the bounds of every read are checked on machines without a GPU.
//
// What is restated: RFC 1950 (zlib container, Adler-32), RFC 1951 (DEFLATE) with the checks zlib's inflate makes, the PNG
// specification's five row filters, and Pillow's convert('RGB') of the modes L, RGB, P, LA and RGBA.
//
// Parallel inflate (after Sitaridi et al., "Massively-parallel lossless data decompression", ICPP 2016, and the block finder of
// Knespel & Brunst, "Rapidgzip", HPDC 2023):
//   1. candidates   every bit offset is tested for a dynamic-Huffman block header that passes full validation (HLIT <= 286,
//                   HDIST <= 30, a complete code-length code, code lengths without a leading repeat or an overrun, complete
//                   literal/length and distance codes or a single distance code, code 256 present), every byte for the
//                   LEN == ~NLEN of a stored block (marking the bit offsets whose 3-bit header would pad to that byte)
//   2. speculative  one thread per subsequence of kSubBytes decodes the block of each of its candidates (up to kSlots) and
//                   records where it ends, how many bytes it inflates to and whether it is the last one
//   3. chain        one thread follows the true block chain from bit 16: where a block start has a clean record it jumps to that
//                   record's end; anywhere else (a fixed-Huffman block, a code a candidate test is stricter about than zlib) it
//                   decodes the block itself.  Every stream completes; one made only of fixed blocks is one sequential decoder.
//                   The running sum of the block lengths is each block's output offset.
//   4. LZ77         one thread per block decodes it again into place: a literal is written, every copied byte gets a pointer
//                   to its source (only stores, so a block's decode never waits on its own output).  Pointer jumping
//                   (src[i] = src[src[i]]) resolves the chains in at most ceil(log2(bytes)) rounds, then every byte is gathered
//                   from its root.  Adler-32 is summed from per-segment partials combined in segment order.
//   5. rows         lane 0 of each of up to kRowWarps warps claims rows in order with an atomic ticket and unfilters them in
//                   place as a wavefront, kRowStep pixels at a time: an Up / Average / Paeth row advances behind the progress
//                   counter of the row above (the filters read left, up and up-left only); None and Sub rows never wait.  The
//                   same pass converts to RGB and stores through the orientation's index map.
// A stream the kernels cannot finish the way zlib + Pillow would (a bad code, a distance too far, a short or long stream,
// trailing data, an Adler-32 mismatch, a filter type above 4, a palette index past the palette) sets bits of the status word,
// and every launch after the chain returns at once when it is set; the caller then decodes that file with Pillow.
#pragma once
#include <stdint.h>

#include "../../include/dust3r_b200.h"

#include "hd.h"

namespace d3r {
namespace png {

constexpr int kSubBytes = 1024;         // stream bytes per speculative-decode thread
constexpr int kSlots = 16;              // block records per subsequence
constexpr int kAdlerSeg = 4096;         // bytes per Adler-32 partial
constexpr int kLitBits = 9;             // direct-lookup bits of the literal/length table
constexpr int kDistBits = 8;            // direct-lookup bits of the distance table
constexpr int kRowWarps = 4096;         // warps of the wavefront (rows in flight); lane 0 of each works
constexpr int kRowStep = 16;            // pixels per chunk of a row: loaded together, then one progress publication

// status word bits
constexpr int kBadCode = D3R_PNG_BAD_CODE, kFar = D3R_PNG_FAR, kShort = D3R_PNG_SHORT, kAdler = D3R_PNG_ADLER,
              kFilter = D3R_PNG_FILTER, kPalette = D3R_PNG_PALETTE;

// order of the code-length code lengths in a dynamic block header
#define D3R_PNG_CLEN_ORDER {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15}
#if defined(__CUDACC__)
__constant__ unsigned char kClenOrderDev[19] = D3R_PNG_CLEN_ORDER;
#endif
static const unsigned char kClenOrderHost[19] = D3R_PNG_CLEN_ORDER;

D3R_HD int clen_order(int i) {
#if defined(__CUDA_ARCH__)
  return kClenOrderDev[i];
#else
  return kClenOrderHost[i];
#endif
}

// Everything the kernels need, derived once from the descriptor on the host (make_plan)
struct Plan {
  int W, H, bpp, color, orientation, palette_len;
  long long n_bytes;                // zlib stream
  long long row_bytes;              // 1 + W * bpp (filter byte + samples)
  long long total;                  // H * row_bytes: what the stream must inflate to
  long long nsub, cap, nseg;        // subsequences, block-chain capacity, Adler segments
  int rounds;                       // pointer-jumping launches
  int out_w, out_h;                 // after the orientation
};

struct Block {                      // one decoded DEFLATE block
  long long start, end;             // bit positions of its header and of the next block's
  long long out_len;                // bytes it inflates to
  int final, err;                   // BFINAL; status bits, 0 when it decoded cleanly
};

struct Link {                       // a block of the true chain
  long long start, out_off;
};

struct Work {                        // workspace pointers
  const d3r_png_desc* desc;
  unsigned long long* ctl;          // [4]: blocks in the chain, bytes inflated, stored Adler-32, row ticket
  int* changed;                     // [rounds] a pointer moved in that round
  int* nrec;                        // [nsub]
  int* progress;                    // [H] pixels of each row unfiltered and stored
  uint32_t* cand;                   // [n_bytes / 4 + 1] bit b of word i: bit offset 32 i + b is a candidate block start
  Block* rec;                       // [nsub][kSlots]
  Link* chain;                      // [cap]
  unsigned long long* adler;        // [nseg] (s1, s2 << 32) of each segment
  int* src;                         // [total] root of each inflated byte (itself for a literal)
  uint8_t* raw;                     // [total] inflated rows, unfiltered in place
  const uint8_t* z;                 // zlib stream
  uint8_t* out;                     // [out_h][out_w][3]
  int* status;
};

D3R_HD void flag(int* status, int bit) {
#if defined(__CUDA_ARCH__)
  atomicOr(status, bit);
#else
  *status |= bit;
#endif
}

D3R_HD int status_of(const Work& w) {
#if defined(__CUDA_ARCH__)
  return *(volatile int*)w.status;
#else
  return *w.status;
#endif
}

// ------------------------------------------------------------------------------------------------ bit reader
// LSB-first, as DEFLATE packs its fields; bytes past the stream read as zero and `over` tells whether any were consumed.
struct Bits {
  const uint8_t* d;
  long long n, next;                // stream bytes, next byte to load
  uint64_t buf;
  int cnt;
  D3R_HD void init(const uint8_t* data, long long n_bytes, long long bit) {
    d = data;
    n = n_bytes;
    next = bit >> 3;
    buf = 0;
    cnt = 0;
    refill();
    drop((int)(bit & 7));
  }
  D3R_HD void refill() {
    if (cnt > 56) return;
    if (next >= 0 && next + 8 <= n) {                         // whole bytes that fit, from eight independent loads
      uint64_t v = 0;
      for (int k = 0; k < 8; ++k) v |= (uint64_t)d[next + k] << (8 * k);
      const int take = (64 - cnt) >> 3;
      if (take < 8) v &= (1ull << (8 * take)) - 1;
      buf |= v << cnt;
      next += take;
      cnt += 8 * take;
      return;
    }
    while (cnt <= 56) {
      buf |= (uint64_t)(next >= 0 && next < n ? d[next] : 0) << cnt;
      ++next;
      cnt += 8;
    }
  }
  D3R_HD unsigned peek(int k) const { return (unsigned)(buf & ((1ull << k) - 1)); }
  D3R_HD void drop(int k) {
    buf >>= k;
    cnt -= k;
  }
  D3R_HD unsigned get(int k) {      // k <= 32
    refill();
    const unsigned v = peek(k);
    drop(k);
    return v;
  }
  D3R_HD long long pos() const { return next * 8 - cnt; }
  D3R_HD bool over() const { return pos() > n * 8; }
};

// ------------------------------------------------------------------------------------------------ Huffman codes
// Kraft sum of n code lengths (0 = unused): 0 complete, 1 a single code of length 1 (the only incomplete code zlib accepts for
// literal/length and distance codes), 2 no code at all, -1 over-subscribed, -2 incomplete otherwise.
D3R_HD int kraft(const uint8_t* len, int n, uint16_t* count) {
  for (int l = 0; l < 16; ++l) count[l] = 0;
  for (int i = 0; i < n; ++i) count[len[i]]++;
  if (count[0] == n) return 2;
  int left = 1, max = 0;
  for (int l = 1; l < 16; ++l) {
    left <<= 1;
    left -= count[l];
    if (left < 0) return -1;
    if (count[l]) max = l;
  }
  if (left == 0) return 0;
  return max == 1 ? 1 : -2;
}

// Canonical decoding table: codes up to B bits by direct lookup ((symbol << 4) | length, 0 = longer or none), longer ones by
// walking the counts.
template <int B, int N>
struct Huff {
  uint16_t fast[1 << B];
  uint16_t count[16];
  uint16_t sym[N];
};

D3R_HD unsigned reverse_bits(unsigned c, int l) {
  unsigned r = 0;
  for (int i = 0; i < l; ++i) r |= ((c >> i) & 1u) << (l - 1 - i);
  return r;
}

template <int B, int N>
D3R_HD int build(Huff<B, N>& h, const uint8_t* len, int n) {
  const int k = kraft(len, n, h.count);
  if (k < 0) return k;
  uint16_t offs[16];
  offs[1] = 0;
  for (int l = 1; l < 15; ++l) offs[l + 1] = (uint16_t)(offs[l] + h.count[l]);
  for (int i = 0; i < n; ++i)
    if (len[i]) h.sym[offs[len[i]]++] = (uint16_t)i;
  for (int i = 0; i < (1 << B); ++i) h.fast[i] = 0;
  unsigned code = 0;
  int idx = 0;
  for (int l = 1; l <= B; ++l) {
    for (int j = 0; j < h.count[l]; ++j, ++idx, ++code) {
      const uint16_t e = (uint16_t)((h.sym[idx] << 4) | l);
      for (unsigned r = reverse_bits(code, l); r < (1u << B); r += 1u << l) h.fast[r] = e;
    }
    code <<= 1;
  }
  return k;
}

// next symbol, or -1 where no code matches
template <int B, int N>
D3R_HD int decode_sym(Bits& b, const Huff<B, N>& h) {
  b.refill();
  const unsigned e = h.fast[b.peek(B)];
  if (e) {
    b.drop((int)(e & 15));
    return (int)(e >> 4);
  }
  int code = 0, first = 0, index = 0;
  for (int l = 1; l < 16; ++l) {
    code |= (int)((b.buf >> (l - 1)) & 1);
    const int c = h.count[l];
    if (code - c < first) {
      b.drop(l);
      return h.sym[index + (code - first)];
    }
    index += c;
    first += c;
    first <<= 1;
    code <<= 1;
  }
  return -1;
}

typedef Huff<kLitBits, 288> LitHuff;
typedef Huff<kDistBits, 32> DistHuff;
typedef Huff<7, 19> ClenHuff;

// Reads a dynamic block header from HLIT on into lens[0, nlit + ndist); 0, or kBadCode where zlib's inflate would stop.
D3R_HD int read_dynamic(Bits& b, uint8_t* lens, int& nlit, int& ndist) {
  nlit = (int)b.get(5) + 257;
  ndist = (int)b.get(5) + 1;
  const int ncode = (int)b.get(4) + 4;
  if (nlit > 286 || ndist > 30) return kBadCode;
  uint8_t cl[19];
  for (int i = 0; i < 19; ++i) cl[i] = 0;
  for (int i = 0; i < ncode; ++i) cl[clen_order(i)] = (uint8_t)b.get(3);
  ClenHuff h;
  if (build(h, cl, 19) != 0) return kBadCode;              // the code-length code must be complete
  const int n = nlit + ndist;
  int i = 0;
  while (i < n) {
    const int s = decode_sym(b, h);
    if (s < 0) return kBadCode;
    if (s < 16) {
      lens[i++] = (uint8_t)s;
      continue;
    }
    int rep;
    uint8_t v = 0;
    if (s == 16) {
      if (i == 0) return kBadCode;                          // repeat with no previous length
      v = lens[i - 1];
      rep = 3 + (int)b.get(2);
    } else if (s == 17) {
      rep = 3 + (int)b.get(3);
    } else {
      rep = 11 + (int)b.get(7);
    }
    if (i + rep > n) return kBadCode;
    while (rep--) lens[i++] = v;
  }
  if (lens[256] == 0) return kBadCode;                      // no end-of-block code
  return 0;
}

// Inflated-byte sink of the write pass: the block's bytes go to raw[base, ...), their roots to src.
struct Sink {
  uint8_t* raw;
  int* src;
  long long base, total;
  int* status;
};

D3R_HD long long length_base(int i, int& extra) {   // literal/length symbol 257 + i
  if (i < 8) {
    extra = 0;
    return 3 + i;
  }
  if (i == 28) {
    extra = 0;
    return 258;
  }
  extra = (i - 4) >> 2;
  return ((long long)(4 + (i & 3)) << extra) + 3;
}

D3R_HD long long dist_base(int d, int& extra) {
  if (d < 4) {
    extra = 0;
    return d + 1;
  }
  extra = (d >> 1) - 1;
  return ((long long)(2 + (d & 1)) << extra) + 1;
}

// Decodes the block whose 3-bit header starts at bit p.  Without a sink it only measures (end, length, last-block flag, errors);
// `limit` bounds the length (a block inflating to more than the image cannot be part of a valid stream).
D3R_HD Block inflate_block(const uint8_t* z, long long n, long long p, long long limit, const Sink* sink) {
  Block r{p, p, 0, 0, 0};
  Bits b;
  b.init(z, n, p);
  r.final = (int)b.get(1);
  const int type = (int)b.get(2);
  if (type == 0) {                                            // stored
    const long long q = (p + 3 + 7) >> 3;
    if (q + 4 > n) {
      r.err = kShort;
      return r;
    }
    const unsigned len = z[q] | (unsigned)z[q + 1] << 8, nlen = z[q + 2] | (unsigned)z[q + 3] << 8;
    if (len != (~nlen & 0xffffu)) {
      r.err = kBadCode;
      return r;
    }
    if (q + 4 + len > n) {
      r.err = kShort;
      return r;
    }
    if (len > limit) {
      r.err = kShort;
      return r;
    }
    if (sink) {
      for (unsigned k = 0; k < len; ++k) {
        const long long o = sink->base + k;
        if (o < sink->total) {
          sink->raw[o] = z[q + 4 + k];
          sink->src[o] = (int)o;
        }
      }
    }
    r.out_len = len;
    r.end = (q + 4 + len) * 8;
    return r;
  }
  if (type == 3) {
    r.err = kBadCode;
    return r;
  }
  LitHuff lit;
  DistHuff dist;
  uint8_t lens[320];
  if (type == 1) {                                            // fixed codes (all 288 / 32 symbols, as zlib builds them)
    for (int i = 0; i < 288; ++i) lens[i] = (uint8_t)(i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8);
    build(lit, lens, 288);
    for (int i = 0; i < 32; ++i) lens[i] = 5;
    build(dist, lens, 32);
  } else {
    int nlit, ndist;
    if (read_dynamic(b, lens, nlit, ndist) || build(lit, lens, nlit) < 0 || build(dist, lens + nlit, ndist) < 0) {
      r.err = b.over() ? kShort : kBadCode;
      return r;
    }
  }
  long long o = 0;
  for (;;) {
    const int s = decode_sym(b, lit);
    if (b.over()) {
      r.err = kShort;
      break;
    }
    if (s < 0 || s >= 286) {
      r.err = kBadCode;
      break;
    }
    if (s < 256) {
      if (o >= limit) {
        r.err = kShort;
        break;
      }
      if (sink && sink->base + o < sink->total) {
        const long long at = sink->base + o;
        sink->raw[at] = (uint8_t)s;
        sink->src[at] = (int)at;
      }
      ++o;
      continue;
    }
    if (s == 256) break;
    int le, de;
    const long long len = length_base(s - 257, le) + b.get(le);
    const int ds = decode_sym(b, dist);
    if (ds < 0 || ds >= 30) {
      r.err = b.over() ? kShort : kBadCode;
      break;
    }
    const long long d = dist_base(ds, de) + b.get(de);
    if (b.over()) {
      r.err = kShort;
      break;
    }
    if (o + len > limit) {
      r.err = kShort;
      break;
    }
    if (sink) {
      for (long long k = 0; k < len; ++k) {
        const long long at = sink->base + o + k, from = at - d;
        if (at >= sink->total) break;
        if (from < 0) {                                       // before the first byte of the stream
          flag(sink->status, kFar);
          sink->src[at] = (int)at;
        } else {                                              // a pointer, resolved by the jumping rounds
          sink->src[at] = (int)from;
        }
      }
    }
    o += len;
  }
  r.out_len = o;
  r.end = b.pos();
  return r;
}

// Header bits BFINAL, BTYPE = 2, HLIT <= 29, HDIST <= 29: the cheap first test of a candidate
D3R_HD bool dynamic_head(unsigned head) {
  return ((head >> 1) & 3) == 2 && ((head >> 3) & 31) <= 29 && ((head >> 8) & 31) <= 29;
}

// Full candidate test for a dynamic block header at bit p whose first 13 bits passed dynamic_head (stricter than zlib: both
// codes complete, or one distance code)
D3R_HD bool dynamic_candidate(const uint8_t* z, long long n, long long p) {
  Bits b;
  b.init(z, n, p);
  b.drop(13);
  int kraft_sum = 0;                                          // the code-length code must be complete: sum of 2^-len == 1
  const int ncode = (int)b.get(4) + 4;
  for (int i = 0; i < ncode; ++i) {
    const int l = (int)b.get(3);
    if (l) kraft_sum += 128 >> l;
  }
  if (kraft_sum != 128) return false;
  b.init(z, n, p + 3);
  uint8_t lens[320];
  int nlit, ndist;
  if (read_dynamic(b, lens, nlit, ndist) || b.over()) return false;
  uint16_t count[16];
  if (kraft(lens, nlit, count) != 0) return false;
  const int kd = kraft(lens + nlit, ndist, count);
  return kd == 0 || kd == 1;
}

D3R_HD void mark(uint32_t* cand, long long bit) {
#if defined(__CUDA_ARCH__)
  atomicOr(cand + (bit >> 5), 1u << (bit & 31));
#else
  cand[bit >> 5] |= 1u << (bit & 31);
#endif
}

D3R_HD void atomic_inc(unsigned long long* p, unsigned long long& old) {
#if defined(__CUDA_ARCH__)
  old = atomicAdd(p, 1ull);
#else
  old = (*p)++;
#endif
}

// ------------------------------------------------------------------------------------------------ per-thread bodies
enum Step { kCand, kSpec, kChain, kWrite, kJump, kGather, kAdlerPart, kAdlerSum, kRows };

// thread t = stream byte t: its 8 bit offsets as dynamic headers, and t as the LEN of a stored block
D3R_HD void cand_body(long long t, const Plan& P, Work& w) {
  if (t >= P.n_bytes) return;
  unsigned win = 0;
  for (int i = 0; i < 3; ++i) win |= (unsigned)(t + i < P.n_bytes ? w.z[t + i] : 0) << (8 * i);
  for (int k = 0; k < 8; ++k)
    if (dynamic_head(win >> k) && dynamic_candidate(w.z, P.n_bytes, 8 * t + k)) mark(w.cand, 8 * t + k);
  if (t + 4 <= P.n_bytes && t >= 1) {
    const unsigned len = w.z[t] | (unsigned)w.z[t + 1] << 8, nlen = w.z[t + 2] | (unsigned)w.z[t + 3] << 8;
    if (len == (~nlen & 0xffffu)) {
      for (long long p = 8 * t - 10; p <= 8 * t - 3; ++p) {
        if (p < 0) continue;
        const unsigned type = (w.z[(p + 1) >> 3] >> ((p + 1) & 7) & 1) | (w.z[(p + 2) >> 3] >> ((p + 2) & 7) & 1) << 1;
        if (type == 0) mark(w.cand, p);
      }
    }
  }
}

// thread t = subsequence t: the block of every candidate in it, in stream order, up to kSlots
D3R_HD void spec_body(long long t, const Plan& P, Work& w) {
  if (t >= P.nsub) return;
  const long long w0 = t * (kSubBytes / 4), w1 = w0 + kSubBytes / 4 < P.n_bytes / 4 + 1 ? w0 + kSubBytes / 4 : P.n_bytes / 4 + 1;
  int k = 0;
  for (long long i = w0; i < w1 && k < kSlots; ++i) {
    uint32_t m = w.cand[i];
    while (m && k < kSlots) {
      int bit = 0;
      while (!((m >> bit) & 1)) ++bit;
      m &= m - 1;
      w.rec[t * kSlots + k++] = inflate_block(w.z, P.n_bytes, i * 32 + bit, P.total, nullptr);
    }
  }
  w.nrec[t] = k;
}

// one thread: the true block chain from bit 16, each block's output offset, the zlib trailer
D3R_HD void chain_body(long long t, const Plan& P, Work& w) {
  if (t != 0) return;
  long long p = 16, off = 0, nb = 0;
  int err = 0;
  for (;;) {
    Block blk;
    bool found = false;
    const long long s = p / (8ll * kSubBytes);
    if (s < P.nsub) {
      for (int j = 0; j < w.nrec[s] && !found; ++j) {
        const Block& r = w.rec[s * kSlots + j];
        if (r.start == p && r.err == 0) {
          blk = r;
          found = true;
        }
      }
    }
    if (!found) blk = inflate_block(w.z, P.n_bytes, p, P.total - off, nullptr);
    if (blk.err) {
      err |= blk.err;
      break;
    }
    if (nb == P.cap || off + blk.out_len > P.total) {
      err |= kShort;
      break;
    }
    w.chain[nb++] = Link{p, off};
    off += blk.out_len;
    p = blk.end;
    if (blk.final) {
      const long long a = (p + 7) >> 3;
      if (a + 4 != P.n_bytes) {
        err |= kShort;                                        // no room for the Adler-32, or data after it
      } else {
        w.ctl[2] = (unsigned long long)w.z[a] << 24 | (unsigned long long)w.z[a + 1] << 16 |
                   (unsigned long long)w.z[a + 2] << 8 | w.z[a + 3];
      }
      break;
    }
  }
  if (off != P.total) err |= kShort;
  if (err) flag(w.status, err);
  w.ctl[0] = (unsigned long long)nb;
  w.ctl[1] = (unsigned long long)off;
}

// thread t = block t of the chain, decoded into place
D3R_HD void write_body(long long t, const Plan& P, Work& w) {
  if (t >= (long long)w.ctl[0] || status_of(w)) return;
  const Link l = w.chain[t];
  Sink k{w.raw, w.src, l.out_off, P.total, w.status};
  inflate_block(w.z, P.n_bytes, l.start, P.total - l.out_off, &k);
}

// round k of pointer jumping, in place (a concurrent update only ever shortens the path a thread reads)
D3R_HD void jump_body(long long t, int k, const Plan& P, Work& w) {
  if (t >= P.total || status_of(w)) return;
  if (k > 0 && w.changed[k - 1] == 0) return;
  const int s = w.src[t];
  if (s == (int)t) return;
  const int r = w.src[s];
  if (r == s) return;
  w.src[t] = r;
  w.changed[k] = 1;
}

D3R_HD void gather_body(long long t, const Plan& P, Work& w) {
  if (t >= P.total || status_of(w)) return;
  const int s = w.src[t];
  if (s != (int)t) w.raw[t] = w.raw[s];
}

constexpr unsigned kAdlerMod = 65521;

// thread t = segment t: (sum of bytes, sum of (bytes left in the segment) * byte), both mod 65521
D3R_HD void adler_part_body(long long t, const Plan& P, Work& w) {
  if (t >= P.nseg || status_of(w)) return;
  const long long b = t * kAdlerSeg, e = b + kAdlerSeg < P.total ? b + kAdlerSeg : P.total;
  unsigned long long s1 = 0, s2 = 0;
  for (long long i = b; i < e; ++i) {
    s1 += w.raw[i];
    s2 += (unsigned long long)(e - i) * w.raw[i];
  }
  w.adler[t] = (s1 % kAdlerMod) | (s2 % kAdlerMod) << 32;
}

D3R_HD void adler_sum_body(long long t, const Plan& P, Work& w) {
  if (t != 0 || status_of(w)) return;
  unsigned long long a = 1, b = 0;
  for (long long s = 0; s < P.nseg; ++s) {
    const long long len = s + 1 < P.nseg ? kAdlerSeg : P.total - s * kAdlerSeg;
    const unsigned long long v = w.adler[s];
    b = (b + (unsigned long long)len * a + (v >> 32)) % kAdlerMod;
    a = (a + (v & 0xffffffffull)) % kAdlerMod;
  }
  if (((b << 16) | a) != w.ctl[2]) flag(w.status, kAdler);
}

D3R_HD int wait_progress(const int* p, int need) {
#if defined(__CUDA_ARCH__)
  int v;
  while ((v = *(const volatile int*)p) < need) __nanosleep(64);
  __threadfence();
  return v;
#else
  (void)need;
  return *p;
#endif
}

D3R_HD void publish(int* p, int v) {
#if defined(__CUDA_ARCH__)
  __threadfence();
  *(volatile int*)p = v;
#else
  *p = v;
#endif
}

D3R_HD uint8_t load_above(const uint8_t* p) {      // a byte another thread unfiltered: read past L1
#if defined(__CUDA_ARCH__)
  return __ldcg(p);
#else
  return *p;
#endif
}

D3R_HD int paeth(int a, int b, int c) {
  const int p = a + b - c;
  const int pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
  if (pa <= pb && pa <= pc) return a;
  return pb <= pc ? b : c;
}

D3R_HD int orient_index(const Plan& P, int x, int y, int& oy) {
  const int W = P.W, H = P.H;
  int ox = x;
  oy = y;
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
  return ox;
}

// Unfilters row y in place (BPP bytes per pixel) in chunks of kRowStep pixels: a chunk's bytes and the bytes above it are
// loaded together, unfiltered from registers, converted to RGB and stored at their oriented places, then the row's progress is
// published.  Only Up, Average and Paeth rows read the row above, so only they wait for it.
template <int BPP>
D3R_HD void unfilter_row(long long y, const Plan& P, Work& w) {
  uint8_t* cur = w.raw + y * P.row_bytes + 1;
  const int f = cur[-1];
  const uint8_t* up = y > 0 ? cur - P.row_bytes : nullptr;
  const int W = P.W;
  if (f > 4) {
    flag(w.status, kFilter);
    publish(w.progress + y, W);
    return;
  }
  const bool reads_up = up && f >= 2;
  int left[BPP], upleft[BPP];
  for (int c = 0; c < BPP; ++c) left[c] = upleft[c] = 0;
  int ready = 0;
  for (int x0 = 0; x0 < W; x0 += kRowStep) {
    const int nx = W - x0 < kRowStep ? W - x0 : kRowStep;
    if (reads_up && x0 + nx > ready) ready = wait_progress(w.progress + y - 1, x0 + nx);
    const long long base = (long long)x0 * BPP;
    int a[kRowStep * BPP], b[kRowStep * BPP];
D3R_UNROLL
    for (int i = 0; i < kRowStep * BPP; ++i) {
      a[i] = i < nx * BPP ? cur[base + i] : 0;
      b[i] = reads_up && i < nx * BPP ? load_above(up + base + i) : 0;
    }
D3R_UNROLL
    for (int px = 0; px < kRowStep; ++px) {
D3R_UNROLL
      for (int c = 0; c < BPP; ++c) {
        const int i = px * BPP + c;
        int v = a[i];
        if (f == 1) v += left[c];
        else if (f == 2) v += b[i];
        else if (f == 3) v += (left[c] + b[i]) >> 1;
        else if (f == 4) v += paeth(left[c], b[i], upleft[c]);
        v &= 255;
        a[i] = v;
        left[c] = v;
        upleft[c] = b[i];
      }
    }
D3R_UNROLL
    for (int px = 0; px < kRowStep; ++px) {
      if (px >= nx) break;
      const int x = x0 + px;
D3R_UNROLL
      for (int c = 0; c < BPP; ++c) cur[base + px * BPP + c] = (uint8_t)a[px * BPP + c];
      int R, G, B;
      if (P.color == 3) {
        const int idx = a[px * BPP];
        if (idx >= P.palette_len) {
          flag(w.status, kPalette);
          R = G = B = 0;
        } else {
          R = w.desc->palette[idx][0];
          G = w.desc->palette[idx][1];
          B = w.desc->palette[idx][2];
        }
      } else if (BPP >= 3) {
        R = a[px * BPP];
        G = a[px * BPP + (BPP >= 3 ? 1 : 0)];
        B = a[px * BPP + (BPP >= 3 ? 2 : 0)];
      } else {
        R = G = B = a[px * BPP];
      }
      int oy;
      const int ox = orient_index(P, x, (int)y, oy);
      uint8_t* o = w.out + ((long long)oy * P.out_w + ox) * 3;
      o[0] = (uint8_t)R;
      o[1] = (uint8_t)G;
      o[2] = (uint8_t)B;
    }
    publish(w.progress + y, x0 + nx);
  }
}

// wavefront: lane 0 of every warp claims rows in order (the row above was claimed by a warp that is already running, so every
// wait ends) and works through them; the other lanes leave at once, so no lane spins against another of its own warp
D3R_HD void rows_body(long long t, const Plan& P, Work& w) {
  if ((t & 31) || (t >> 5) >= kRowWarps || status_of(w)) return;
  for (;;) {
    unsigned long long y;
    atomic_inc(w.ctl + 3, y);
    if (y >= (unsigned long long)P.H) return;
    if (P.bpp == 1) unfilter_row<1>((long long)y, P, w);
    else if (P.bpp == 2) unfilter_row<2>((long long)y, P, w);
    else if (P.bpp == 3) unfilter_row<3>((long long)y, P, w);
    else unfilter_row<4>((long long)y, P, w);
  }
}

template <int S>
D3R_HD void step(long long t, int k, const Plan& P, Work& w) {
  if (S == kCand) cand_body(t, P, w);
  else if (S == kSpec) spec_body(t, P, w);
  else if (S == kChain) chain_body(t, P, w);
  else if (S == kWrite) write_body(t, P, w);
  else if (S == kJump) jump_body(t, k, P, w);
  else if (S == kGather) gather_body(t, P, w);
  else if (S == kAdlerPart) adler_part_body(t, P, w);
  else if (S == kAdlerSum) adler_sum_body(t, P, w);
  else rows_body(t, P, w);
}

// ------------------------------------------------------------------------------------------------ host side
inline long long align_up(long long b) { return (b + 255) / 256 * 256; }

// Plan of a descriptor, or an error message (argument checks before any launch)
inline const char* make_plan(const d3r_png_desc& D, long long n_bytes, Plan& P) {
  P = Plan{};
  if (D.width < 1 || D.height < 1) return "image size below 1";
  if (D.orientation < 1 || D.orientation > 8) return "orientation outside [1, 8]";
  int bpp;
  switch (D.color_type) {
    case 0: bpp = 1; break;
    case 2: bpp = 3; break;
    case 3: bpp = 1; break;
    case 4: bpp = 2; break;
    case 6: bpp = 4; break;
    default: return "colour type outside {0, 2, 3, 4, 6}";
  }
  if (D.color_type == 3 ? (D.palette_len < 1 || D.palette_len > 256) : D.palette_len != 0)
    return "palette length outside [1, 256] for colour type 3, or a palette for another colour type";
  if (n_bytes < 6 || n_bytes != D.idat_bytes) return "stream byte count below 6 or not idat_bytes";
  P.W = D.width;
  P.H = D.height;
  P.bpp = bpp;
  P.color = D.color_type;
  P.orientation = D.orientation;
  P.palette_len = D.palette_len;
  P.n_bytes = n_bytes;
  P.row_bytes = 1 + (long long)P.W * bpp;
  P.total = P.row_bytes * P.H;
  if (P.total >= (1ll << 31) - 1) return "image rows of 2^31 bytes or more";
  P.nsub = (n_bytes + kSubBytes - 1) / kSubBytes;
  P.cap = n_bytes / 16 + 64;
  P.nseg = (P.total + kAdlerSeg - 1) / kAdlerSeg;
  int r = 1;
  while ((1ll << (r - 1)) < P.total) ++r;
  P.rounds = r + 1;                                           // ceil(log2(total)) rounds, and one that sees no change
  const bool swap = P.orientation >= 5;
  P.out_w = swap ? P.H : P.W;
  P.out_h = swap ? P.W : P.H;
  return nullptr;
}

// workspace: [desc][ctl][changed][nrec][progress][cand][rec][chain][adler][src][raw], each 256-byte aligned; the first five
// after desc are zeroed by each call
struct Layout {
  long long desc, ctl, changed, nrec, progress, cand, rec, chain, adler, src, raw, bytes;
  explicit Layout(const Plan& P) {
    desc = 0;
    ctl = desc + align_up(sizeof(d3r_png_desc));
    changed = ctl + align_up(32);
    nrec = changed + align_up(4ll * P.rounds);
    progress = nrec + align_up(4 * P.nsub);
    cand = progress + align_up(4ll * P.H);
    rec = cand + align_up(4 * (P.n_bytes / 4 + 1));
    chain = rec + align_up((long long)sizeof(Block) * kSlots * P.nsub);
    adler = chain + align_up((long long)sizeof(Link) * P.cap);
    src = adler + align_up(8 * P.nseg);
    raw = src + align_up(4 * P.total);
    bytes = raw + align_up(P.total);
  }
  Work work(char* ws) const {
    Work w{};
    w.desc = reinterpret_cast<const d3r_png_desc*>(ws + desc);
    w.ctl = reinterpret_cast<unsigned long long*>(ws + ctl);
    w.changed = reinterpret_cast<int*>(ws + changed);
    w.nrec = reinterpret_cast<int*>(ws + nrec);
    w.progress = reinterpret_cast<int*>(ws + progress);
    w.cand = reinterpret_cast<uint32_t*>(ws + cand);
    w.rec = reinterpret_cast<Block*>(ws + rec);
    w.chain = reinterpret_cast<Link*>(ws + chain);
    w.adler = reinterpret_cast<unsigned long long*>(ws + adler);
    w.src = reinterpret_cast<int*>(ws + src);
    w.raw = reinterpret_cast<uint8_t*>(ws + raw);
    return w;
  }
};

// The launch sequence, shared by the CUDA entry point and the host harness.  L provides
//   zero(ptr, bytes), copy_desc(dst, src), and template <int S> launch(n_threads, k, plan, work).
template <class L>
void decode(L& l, const Plan& P, const Layout& lay, Work& w, const d3r_png_desc& desc, char* ws) {
  l.copy_desc(ws + lay.desc, &desc);
  l.zero(w.status, 4);
  l.zero(ws + lay.ctl, lay.rec - lay.ctl);                  // control words, round flags, record counts, row progress, candidates
  l.template launch<kCand>(P.n_bytes, 0, P, w);
  l.template launch<kSpec>(P.nsub, 0, P, w);
  l.template launch<kChain>(1, 0, P, w);
  l.template launch<kWrite>(P.cap, 0, P, w);
  for (int k = 0; k < P.rounds; ++k) l.template launch<kJump>(P.total, k, P, w);
  l.template launch<kGather>(P.total, 0, P, w);
  l.template launch<kAdlerPart>(P.nseg, 0, P, w);
  l.template launch<kAdlerSum>(1, 0, P, w);
  l.template launch<kRows>(32ll * (P.H < kRowWarps ? P.H : kRowWarps), 0, P, w);
}

// What the step-decoder launchers (csrc/step_decode.cuh, tests/native/step_host.h) need of this codec
struct Codec {
  using Desc = d3r_png_desc;
  using Plan = png::Plan;
  using Work = png::Work;
  using Layout = png::Layout;
  static constexpr const char* kEntry = "d3r_png_decode";
  static constexpr const char* kTag = "png_decode";
  static constexpr const uint8_t* Work::*kInput = &Work::z;
  static const char* make_plan(const Desc& D, long long n_bytes, Plan& P) { return png::make_plan(D, n_bytes, P); }
  template <class L>
  static void decode(L& l, const Plan& P, const Layout& lay, Work& w, const Desc& desc, char* ws) {
    png::decode(l, P, lay, w, desc, ws);
  }
  template <int S>
  D3R_HD static void step(long long t, int k, const Plan& P, Work& w) { png::step<S>(t, k, P, w); }
  // compulsory traffic: the stream (read about three times), the inflated rows and their roots written, read and written
  // again, the RGB out
  static double traffic(const Plan& P, long long n_bytes) {
    return 3.0 * double(n_bytes) + 4.0 * double(P.total) + 8.0 * double(P.total) + 3.0 * double(P.W) * P.H;
  }
  static int launches(const Plan& P) { return P.rounds + 8; }
};

}  // namespace png
}  // namespace d3r
