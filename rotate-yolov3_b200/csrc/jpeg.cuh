// The per-symbol and per-pixel arithmetic of the JPEG decoder (csrc/jpeg.cu), as __host__ __device__ functions so that a
// host build of the same code can be checked against cv2.imread without a GPU (tests/test_jpeg_cpu.py).  Each function
// restates what libjpeg-turbo 3.1's default decompression computes:
//
//   entropy    jdhuff.c decode_mcu: canonical Huffman codes (HUFF_DECODE), HUFF_EXTEND of the extra bits, (run, size)
//              AC symbols with EOB and ZRL; 0xFF00 byte stuffing is skipped by the bit reader.  Reads past the end of
//              a segment see zero bits, as libjpeg's fill_bit_buffer supplies them.
//   IDCT       jidctint.c jpeg_idct_islow: 13-bit constants, PASS1_BITS 2, 64-bit products, rounding descale, the
//              output plus 128 saturated; a block outside the range where that equals every libjpeg-turbo IDCT gets
//              RYOLO_JPEG_ST_RANGE (idct_islow below).
//   upsample   jdsample.c: h2v1 / h2v2 fancy (triangle) upsampling when the component is wider than 2 samples
//              (box replication otherwise), h1v2 fancy, 4:1:1 box; first / last column replicated; context rows
//              replicated at the top and at the last real row (jdmainct.c set_bottom_pointers).
//   colour     jdcolor.c ycc_rgb_convert with its SCALEBITS 16 tables, stored B, G, R; gray replicated; RGB reordered.
//   orientation  cv2's ExifTransform (flip / transpose) as a map from an output pixel to a stored pixel.
#pragma once
#include <stdint.h>

#include "../../include/ryolo.h"

#ifdef __CUDACC__
#define RJ_HD __host__ __device__ __forceinline__
#else
#define RJ_HD inline
#endif

namespace ryolo {
namespace jpeg {

// A thread that has not synchronised after this many chunks and this many bytes gives up.  A decoder on the right symbol
// boundaries can still be at the wrong block of the MCU, decoding with another component's tables; at high quality few
// blocks end in an EOB and it may take a few kilobytes to fall onto the true state.
constexpr int kMaxSyncChunks = 32;
constexpr int kMaxSyncBytes = 16384;

#ifdef __CUDACC__
__constant__ uint8_t kNaturalDev[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
#endif
static const uint8_t kNaturalHost[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// position of the k-th coefficient in zigzag order within the 8x8 block (jpeg_natural_order)
RJ_HD int natural(int k) {
#ifdef __CUDA_ARCH__
  return kNaturalDev[k];
#else
  return kNaturalHost[k];
#endif
}

// ---------------------------------------------------------------------------------------------------------------------
// Entropy decoding
// ---------------------------------------------------------------------------------------------------------------------

// A decoder state: the next unread bit (byte, bit; byte never points at the 0x00 of a stuffed 0xFF00), the zigzag index
// of the next coefficient of the current block (0: its DC) and the block within the MCU.
struct State {
  uint32_t byte, bit, z, blk;
};
RJ_HD bool same(const State& a, const State& b) {
  return a.byte == b.byte && a.bit == b.bit && a.z == b.z && a.blk == b.blk;
}
// two words per state in the workspace
RJ_HD void pack(const State& s, uint32_t* w) {
  w[0] = s.byte;
  w[1] = s.bit | (s.z << 3) | (s.blk << 10);
}
RJ_HD State unpack(const uint32_t* w) {
  State s;
  s.byte = w[0], s.bit = w[1] & 7u, s.z = (w[1] >> 3) & 127u, s.blk = w[1] >> 10;
  return s;
}

// 32 bits from (byte, bit) on, skipping stuffed zeros; bytes at or past `end` read as 0
RJ_HD uint32_t peek32(const uint8_t* d, uint32_t end, uint32_t byte, uint32_t bit) {
  uint64_t acc = 0;
  uint32_t i = byte;
#pragma unroll
  for (int j = 0; j < 5; j++) {
    const uint32_t b = i < end ? d[i] : 0u;
    acc = (acc << 8) | b;
    i += b == 0xFFu ? 2u : 1u;
  }
  return (uint32_t)(acc >> (8 - bit));
}

RJ_HD void advance(const uint8_t* d, uint32_t end, State& s, uint32_t n) {
  s.bit += n;
  while (s.bit >= 8) {
    s.bit -= 8;
    s.byte += (s.byte < end && d[s.byte] == 0xFFu) ? 2u : 1u;
  }
}

// the symbol whose code starts at the top of `bits` and its code length; -1 when no code of <= 16 bits matches
RJ_HD int huff_decode(const ryolo_jpeg_huff& h, uint32_t bits, int& len) {
  const uint32_t e = h.lut[bits >> 23];
  if (e) {
    len = (int)(e >> 8);
    return (int)(e & 0xFFu);
  }
  for (int l = 10; l <= 16; l++) {
    const int32_t code = (int32_t)(bits >> (32 - l));
    if (code <= h.maxcode[l]) {
      len = l;
      return h.vals[(code + h.valoff[l]) & 0xFF];
    }
  }
  len = 0;
  return -1;
}

// HUFF_EXTEND: the s-bit magnitude category value r as a signed coefficient
RJ_HD int extend(uint32_t r, int s) { return (int)r < (1 << (s - 1)) ? (int)r - (1 << s) + 1 : (int)r; }

RJ_HD int component_of(const ryolo_jpeg_image& im, uint32_t blk) {
  return blk >= (uint32_t)im.boff[2] ? 2 : blk >= (uint32_t)im.boff[1] ? 1 : 0;
}

// Decodes one symbol at s and advances s.  On success returns true with zpos / value the zigzag position and value of
// the coefficient it sets (zpos = -1 for EOB and ZRL); the symbol covers positions [z before, z after) of its block,
// z after = 64 when the block ends (s.z is then 0 and s.blk the next block).  On a code not in the table, or a run past
// position 63, returns false having advanced one bit and kept z and blk (the rule the speculative chunk decoders
// follow; a decoder on the true path reports it).
RJ_HD bool step(const uint8_t* d, uint32_t end, const ryolo_jpeg_huff* huff, const ryolo_jpeg_image& im, State& s,
                int& zpos, int& value) {
  const int ci = component_of(im, s.blk);
  const uint32_t bits = peek32(d, end, s.byte, s.bit);
  int len = 0;
  if (s.z == 0) {
    const int sz = huff_decode(huff[im.dctab[ci]], bits, len);
    if (sz < 0 || sz > 15) {
      advance(d, end, s, 1);
      return false;
    }
    value = sz ? extend((bits << len) >> (32 - sz), sz) : 0;
    zpos = 0;
    advance(d, end, s, (uint32_t)(len + sz));
    s.z = 1;
  } else {
    const int rs = huff_decode(huff[im.actab[ci]], bits, len);
    if (rs < 0) {
      advance(d, end, s, 1);
      return false;
    }
    const int r = rs >> 4, sz = rs & 15;
    if (sz) {
      const int z = (int)s.z + r;
      if (z > 63) {
        advance(d, end, s, 1);
        return false;
      }
      value = extend((bits << len) >> (32 - sz), sz);
      zpos = z;
      advance(d, end, s, (uint32_t)(len + sz));
      s.z = (uint32_t)z + 1;
    } else if (r == 15) {                                  // ZRL: sixteen zeros
      if (s.z + 16 > 64) {
        advance(d, end, s, 1);
        return false;
      }
      zpos = -1;
      advance(d, end, s, (uint32_t)len);
      s.z += 16;
    } else {                                               // EOB
      zpos = -1;
      advance(d, end, s, (uint32_t)len);
      s.z = 64;
    }
  }
  if (s.z >= 64) {
    s.z = 0;
    s.blk = s.blk + 1 == (uint32_t)im.bpm ? 0u : s.blk + 1;
  }
  return true;
}

// first byte of chunk k of a segment (k = nchunk: the segment end); a chunk never starts on a stuffed zero
RJ_HD uint32_t chunk_start(const uint8_t* d, const ryolo_jpeg_segment& sg, int k, int chunk_bytes) {
  if (k <= 0) return (uint32_t)sg.start;
  const int64_t b64 = sg.start + (int64_t)k * chunk_bytes;
  if (k >= sg.nchunk || b64 >= sg.end) return (uint32_t)sg.end;
  uint32_t b = (uint32_t)b64;
  if (b > (uint32_t)sg.start && d[b - 1] == 0xFFu) b++;
  return b;
}

RJ_HD State segment_start(const ryolo_jpeg_segment& sg) {
  State s;
  s.byte = (uint32_t)sg.start, s.bit = 0, s.z = 0, s.blk = 0;
  return s;
}

// Pass A of chunk c (k-th of its segment): decode from the chunk's first byte, as if a block began there, to the first
// symbol boundary at or past the chunk's end.  Returns that state.
RJ_HD State chunk_pass_a(const uint8_t* d, const ryolo_jpeg_segment& sg, const ryolo_jpeg_image& im,
                         const ryolo_jpeg_huff* huff, int k, int chunk_bytes) {
  State s = k == 0 ? segment_start(sg) : State{chunk_start(d, sg, k, chunk_bytes), 0u, 0u, 0u};
  const uint32_t stop = chunk_start(d, sg, k + 1, chunk_bytes), end = (uint32_t)sg.end;
  int zpos, value;
  while (s.byte < stop) step(d, end, huff, im, s, zpos, value);
  return s;
}

// Pass B of chunk k: decode on from `s` (where the previous chunk's pass-A decoder stopped; the segment start for k = 0)
// through chunk k, k + 1, ... until the state at the end of chunk j equals exits[j] (pass A's state there) or j is the
// segment's last chunk.  Returns j, or -1 when that takes more than kMaxSyncChunks chunks and kMaxSyncBytes bytes.  *blocks: blocks begun.
RJ_HD int chunk_pass_b(const uint8_t* d, const ryolo_jpeg_segment& sg, const ryolo_jpeg_image& im,
                       const ryolo_jpeg_huff* huff, int k, int chunk_bytes, State s, const uint32_t* exits,
                       int* blocks) {
  const uint32_t end = (uint32_t)sg.end, start = s.byte;
  int nb = 0, zpos, value;
  for (int j = k; j < sg.nchunk; j++) {
    const uint32_t stop = chunk_start(d, sg, j + 1, chunk_bytes);
    while (s.byte < stop) {
      const uint32_t z0 = s.z;
      if (step(d, end, huff, im, s, zpos, value) && z0 == 0) nb++;
    }
    if (j == sg.nchunk - 1 || same(s, unpack(exits + 2 * j))) {
      *blocks = nb;
      return j;
    }
    if (j - k >= kMaxSyncChunks && stop - start > (uint32_t)kMaxSyncBytes) break;
  }
  *blocks = nb;
  return -1;
}

// The chain rule of the resolve step, over a window of 32 chunks p, p + 1, ... from the chain's current chunk p (the
// kernel takes one window per warp step).  `first` is the first offset i whose pass B did not stop in its own chunk
// (jump[p + i] != p + i; 32 when every chunk of the window did), jump_first that chunk's pass-B result.  Chunk p + i
// is on the chain iff i < first, or i == first and its pass B synchronised (jump_first >= 0): a chunk whose pass B did
// not synchronise gets no writer.  next_chain: the chain's next chunk, or -1 when it breaks (RYOLO_JPEG_ST_NO_SYNC).
RJ_HD bool on_chain(int i, int first, int jump_first) { return i < first || (i == first && jump_first >= 0); }
RJ_HD int next_chain(int p, int first, int jump_first) {
  return first == 32 ? p + 32 : (jump_first < 0 ? -1 : jump_first + 1);
}

// The writer of a chunk on the true decode path: decode from `s` (its true start state) to the end of chunk `last`,
// storing each block's coefficients (natural order; the DC as its difference) into blocks[0 .. nblocks) of the
// segment.  first_block: blocks of the segment begun before s.  Stops after the segment's last block.  Returns 0 or a
// RYOLO_JPEG_ST_* mask.
RJ_HD int chunk_write(const uint8_t* d, const ryolo_jpeg_segment& sg, const ryolo_jpeg_image& im,
                      const ryolo_jpeg_huff* huff, int last, int chunk_bytes, State s, int first_block,
                      int16_t* blocks) {
  if (last < 0 || last >= sg.nchunk) return RYOLO_JPEG_ST_NO_SYNC;     // not on a synchronised chain
  const uint32_t end = (uint32_t)sg.end, stop = chunk_start(d, sg, last + 1, chunk_bytes);
  const int nblocks = sg.nmcu * im.bpm;
  // every block was completed before s (whose writer checked where): the rest is padding after the last block
  if (first_block > nblocks || (first_block == nblocks && s.z == 0)) return 0;
  int cur = first_block - 1, zpos = -1, value = 0;
  bool done = false;
  while (s.byte < stop) {
    if (s.z == 0 && cur + 1 >= nblocks) {
      done = true;
      break;
    }
    const uint32_t z0 = s.z;
    if (!step(d, end, huff, im, s, zpos, value)) return RYOLO_JPEG_ST_BAD_CODE;
    if (z0 == 0) cur++;
    if (cur < 0 || cur >= nblocks) return RYOLO_JPEG_ST_BAD_CODE;
    int16_t* blk = blocks + (int64_t)cur * 64;
    const uint32_t z1 = s.z == 0 ? 64u : s.z;
    for (uint32_t p = z0; p < z1; p++) blk[natural((int)p)] = (int16_t)((int)p == zpos ? value : 0);
  }
  if (!done && s.z == 0 && cur + 1 >= nblocks) done = true;
  if (done) return (s.byte < end || (s.byte == end && s.bit == 0)) ? 0 : RYOLO_JPEG_ST_TRUNCATED;
  return last == sg.nchunk - 1 ? RYOLO_JPEG_ST_TRUNCATED : 0;
}

// the block (decode order, within the image) of the e-th block of component ci in a segment, for the DC prefix: DC
// differences become values by a running sum per component that restarts with every segment (a restart marker).  The
// sum wraps as libjpeg's unsigned int arithmetic does; the block keeps its low 16 bits (JCOEF).
RJ_HD int64_t dc_block(const ryolo_jpeg_image& im, const ryolo_jpeg_segment& sg, int ci, int64_t e) {
  const int n = im.h[ci] * im.v[ci];
  const int64_t m = e / n;
  return ((int64_t)sg.first_mcu + m) * im.bpm + im.boff[ci] + (e - m * n);
}

// ---------------------------------------------------------------------------------------------------------------------
// Dequantisation and the ISLOW IDCT (jidctint.c)
// ---------------------------------------------------------------------------------------------------------------------

// Which IDCT cv2 runs depends on its libjpeg-turbo build: the C jidctint.c (64-bit products, and the output through a
// range-limit table indexed with a 10-bit wrap) or, with SIMD, jidctint-sse2 / -avx2 (dequantisation and both passes'
// inputs and outputs in 16-bit lanes with 32-bit products, the output saturated).  The two compute the same integers,
// and this function computes them too, only while a block stays in the range real 8-bit pixels produce.  A block
// whose dequantised coefficients or output leave it (a corrupt stream, an odd encoder) is decoded differently by the
// two, so idct_islow returns RYOLO_JPEG_ST_RANGE for it and the image goes to the host decoder.  The predicate:
//
//   (a) every column c of dequantised coefficients F[u][c] = coef * q has  2 |F[0][c]| + 3 sum_{u>=1} |F[u][c]| <= 8192
//   (b) every output value x (the pass-2 sum after its descale, before the + 128) lies in [-512, 511].
//
// Why it suffices.  Pass 1 is linear before its rounding: ws[n][c] = (sum_u M[n][u] F[u][c] + 2^10) >> 11, M the 8x8
// integer matrix of the butterflies.  |M[n][0]| = 2^13 and |M[n][u]| <= 11387 = 1.39 * 2^13 for u >= 1 (sqrt 2
// cos(pi / 16) = 1.387; tests/test_jpeg_syntax_cpu.py restates pass 1, builds M and checks both).  With 2 * 1.39 <= 3,
// (a) gives |F[0][c]| + 1.39 sum_{u>=1} |F[u][c]| <= 4096, so
//   |ws[n][c]| <= 4 * 4096 + 1 = 16385,  half of int16,  and every |F| <= 4096,  an eighth of it:
// no 16-bit lane wraps or saturates in dequantisation or pass 1.  Pass 2's sums are at most 8 * 16385 * 11387 <
// 1.5e9, inside int32, so every path holds the same x.  By (b), x + 128 through the 10-bit wrap is x + 128 itself, and
// the table and the SIMD saturation give the same byte.  (b) is needed besides (a): a bound on the coefficients alone
// that implies it (sum of |F| weighted by the IDCT's largest gains, or |F[0][0]| / 8 plus the AC energy) reaches past
// 600 on the noisy q100 test pictures, whose outputs stay inside [-128, 127].
constexpr int kIdctColumnLimit = 8192;
constexpr int kIdctOutMin = -512, kIdctOutMax = 511;

RJ_HD int min_abs(int v, int cap) {
  const int a = v < 0 ? -v : v;
  return a < cap ? a : cap;
}

// the rounding descale of a pass-2 sum; out of [kIdctOutMin, kIdctOutMax] sets *bad.  The descaled value is taken in
// 32 bits: under (a) it is below 1.5e9 / 2^18 in magnitude, and a block breaking (a) is flagged whatever it wraps to.
RJ_HD int descale_out(int64_t x, int shift, bool& bad) {
  const int v = (int)((x + ((int64_t)1 << (shift - 1))) >> shift);
  bad |= (unsigned)(v - kIdctOutMin) > (unsigned)(kIdctOutMax - kIdctOutMin);
  return v < -128 ? 0 : (v > 127 ? 255 : v + 128);
}

// coef: 64 coefficients in natural order, q: the quantisation table in natural order; out: 8 rows of `pitch` bytes.
// Returns 0, or RYOLO_JPEG_ST_RANGE when the block breaks the predicate above (out then holds saturated values).
RJ_HD int idct_islow(const int16_t* coef, const uint16_t* q, uint8_t* out, int pitch) {
  constexpr int CB = 13, P1 = 2;
  int ws[64];
  bool bad = false;
#pragma unroll
  for (int c = 0; c < 8; c++) {
    int64_t z1, z2, z3, z4, z5, t0, t1, t2, t3, t10, t11, t12, t13;
    int f[8];
#pragma unroll
    for (int u = 0; u < 8; u++) f[u] = (int)coef[8 * u + c] * (int)q[8 * u + c];
    // in 32 bits: each |f| capped at the limit (a capped term alone breaks it) keeps the sum below 2^18
    int col = 2 * min_abs(f[0], kIdctColumnLimit);
#pragma unroll
    for (int u = 1; u < 8; u++) col += 3 * min_abs(f[u], kIdctColumnLimit);
    bad |= col > kIdctColumnLimit;
    z2 = f[2], z3 = f[6];
    z1 = (z2 + z3) * 4433;
    t2 = z1 + z3 * -15137;
    t3 = z1 + z2 * 6270;
    z2 = f[0], z3 = f[4];
    t0 = (z2 + z3) * ((int64_t)1 << CB);
    t1 = (z2 - z3) * ((int64_t)1 << CB);
    t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    t0 = f[7], t1 = f[5], t2 = f[3], t3 = f[1];
    z1 = t0 + t3, z2 = t1 + t2, z3 = t0 + t2, z4 = t1 + t3;
    z5 = (z3 + z4) * 9633;
    t0 *= 2446, t1 *= 16819, t2 *= 25172, t3 *= 12299;
    z1 *= -7373, z2 *= -20995, z3 *= -16069, z4 *= -3196;
    z3 += z5, z4 += z5;
    t0 += z1 + z3, t1 += z2 + z4, t2 += z2 + z3, t3 += z1 + z4;
    constexpr int sh = CB - P1;
    constexpr int64_t rnd = (int64_t)1 << (sh - 1);
    ws[c] = (int32_t)((t10 + t3 + rnd) >> sh);
    ws[56 + c] = (int32_t)((t10 - t3 + rnd) >> sh);
    ws[8 + c] = (int32_t)((t11 + t2 + rnd) >> sh);
    ws[48 + c] = (int32_t)((t11 - t2 + rnd) >> sh);
    ws[16 + c] = (int32_t)((t12 + t1 + rnd) >> sh);
    ws[40 + c] = (int32_t)((t12 - t1 + rnd) >> sh);
    ws[24 + c] = (int32_t)((t13 + t0 + rnd) >> sh);
    ws[32 + c] = (int32_t)((t13 - t0 + rnd) >> sh);
  }
#pragma unroll
  for (int r = 0; r < 8; r++) {
    const int* w = ws + 8 * r;
    int64_t z1, z2, z3, z4, z5, t0, t1, t2, t3, t10, t11, t12, t13;
    z2 = w[2], z3 = w[6];
    z1 = (z2 + z3) * 4433;
    t2 = z1 + z3 * -15137;
    t3 = z1 + z2 * 6270;
    t0 = ((int64_t)w[0] + (int64_t)w[4]) * ((int64_t)1 << CB);
    t1 = ((int64_t)w[0] - (int64_t)w[4]) * ((int64_t)1 << CB);
    t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    t0 = w[7], t1 = w[5], t2 = w[3], t3 = w[1];
    z1 = t0 + t3, z2 = t1 + t2, z3 = t0 + t2, z4 = t1 + t3;
    z5 = (z3 + z4) * 9633;
    t0 *= 2446, t1 *= 16819, t2 *= 25172, t3 *= 12299;
    z1 *= -7373, z2 *= -20995, z3 *= -16069, z4 *= -3196;
    z3 += z5, z4 += z5;
    t0 += z1 + z3, t1 += z2 + z4, t2 += z2 + z3, t3 += z1 + z4;
    constexpr int sh = CB + P1 + 3;
    uint8_t* o = out + (int64_t)r * pitch;
    o[0] = (uint8_t)descale_out(t10 + t3, sh, bad);
    o[7] = (uint8_t)descale_out(t10 - t3, sh, bad);
    o[1] = (uint8_t)descale_out(t11 + t2, sh, bad);
    o[6] = (uint8_t)descale_out(t11 - t2, sh, bad);
    o[2] = (uint8_t)descale_out(t12 + t1, sh, bad);
    o[5] = (uint8_t)descale_out(t12 - t1, sh, bad);
    o[3] = (uint8_t)descale_out(t13 + t0, sh, bad);
    o[4] = (uint8_t)descale_out(t13 - t0, sh, bad);
  }
  return bad ? RYOLO_JPEG_ST_RANGE : 0;
}

// plane position of block b (decode order) of an image: component, first row, first column
RJ_HD int block_position(const ryolo_jpeg_image& im, int64_t b, int& row, int& col) {
  const int64_t m = b / im.bpm;
  const int j = (int)(b - m * im.bpm);
  const int ci = component_of(im, (uint32_t)j);
  const int k = j - im.boff[ci];
  const int my = (int)(m / im.mcux), mx = (int)(m - (int64_t)my * im.mcux);
  row = 8 * (my * im.v[ci] + k / im.h[ci]);
  col = 8 * (mx * im.h[ci] + k % im.h[ci]);
  return ci;
}

// ---------------------------------------------------------------------------------------------------------------------
// Upsampling, colour conversion and orientation
// ---------------------------------------------------------------------------------------------------------------------

RJ_HD int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// component ci's sample at stored pixel (x, y), upsampled as jdsample.c does it
RJ_HD int upsample(const ryolo_jpeg_image& im, const uint8_t* plane, int ci, int x, int y) {
  const int rh = im.hmax / im.h[ci], rv = im.vmax / im.v[ci], pitch = im.pitch[ci], dw = im.dw[ci], dh = im.dh[ci];
  if (rh == 1 && rv == 1) return plane[(int64_t)y * pitch + x];
  if (rh == 4 || ((rh == 2) && dw <= 2)) return plane[(int64_t)(y / rv) * pitch + x / rh];   // box replication
  const int j = x / rh, r = y / rv;
  if (rh == 1) {                                       // h1v2: (3 * nearer row + further row + 1 or 2) >> 2
    const int far = (y & 1) ? clampi(r + 1, 0, dh - 1) : clampi(r - 1, 0, dh - 1);
    return (3 * plane[(int64_t)r * pitch + j] + plane[(int64_t)far * pitch + j] + ((y & 1) ? 2 : 1)) >> 2;
  }
  const int jn = (x & 1) ? clampi(j + 1, 0, dw - 1) : clampi(j - 1, 0, dw - 1);
  if (rv == 1) {                                       // h2v1: (3 * nearer + further + 1 or 2) >> 2
    const uint8_t* p = plane + (int64_t)r * pitch;
    return (3 * p[j] + p[jn] + ((x & 1) ? 2 : 1)) >> 2;
  }
  // h2v2: column sums 3 * nearer row + further row, then (3 * nearer sum + further sum + 8 or 7) >> 4
  const int far = (y & 1) ? clampi(r + 1, 0, dh - 1) : clampi(r - 1, 0, dh - 1);
  const uint8_t* p0 = plane + (int64_t)r * pitch;
  const uint8_t* p1 = plane + (int64_t)far * pitch;
  const int c0 = 3 * p0[j] + p1[j], c1 = 3 * p0[jn] + p1[jn];
  return (3 * c0 + c1 + ((x & 1) ? 7 : 8)) >> 4;
}

// stored pixel of output pixel (ox, oy) under Exif orientation o (cv2's flip / transpose sequence)
RJ_HD void orient_source(const ryolo_jpeg_image& im, int ox, int oy, int& x, int& y) {
  const int W = im.width, H = im.height;
  switch (im.orient) {
    case 2: x = W - 1 - ox, y = oy; break;
    case 3: x = W - 1 - ox, y = H - 1 - oy; break;
    case 4: x = ox, y = H - 1 - oy; break;
    case 5: x = oy, y = ox; break;
    case 6: x = oy, y = H - 1 - ox; break;
    case 7: x = W - 1 - oy, y = H - 1 - ox; break;
    case 8: x = W - 1 - oy, y = ox; break;
    default: x = ox, y = oy; break;
  }
}

// output pixel (ox, oy) as B, G, R; planes: the image area
RJ_HD void pixel_bgr(const ryolo_jpeg_image& im, const uint8_t* area, int ox, int oy, uint8_t* bgr) {
  int x, y;
  orient_source(im, ox, oy, x, y);
  const int c0 = upsample(im, area + im.plane_off[0], 0, x, y);
  if (im.color == RYOLO_JPEG_GRAY) {
    bgr[0] = bgr[1] = bgr[2] = (uint8_t)c0;
    return;
  }
  const int c1 = upsample(im, area + im.plane_off[1], 1, x, y);
  const int c2 = upsample(im, area + im.plane_off[2], 2, x, y);
  if (im.color == RYOLO_JPEG_RGB) {
    bgr[0] = (uint8_t)c2, bgr[1] = (uint8_t)c1, bgr[2] = (uint8_t)c0;
    return;
  }
  // jdcolor.c build_ycc_rgb_table: FIX(1.40200) = 91881, FIX(1.77200) = 116130, FIX(0.71414) = 46802,
  // FIX(0.34414) = 22554, ONE_HALF = 1 << 15; right shifts are arithmetic
  const int cb = c1 - 128, cr = c2 - 128;
  const int r = c0 + ((91881 * cr + 32768) >> 16);
  const int g = c0 + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
  const int b = c0 + ((116130 * cb + 32768) >> 16);
  bgr[0] = (uint8_t)clampi(b, 0, 255), bgr[1] = (uint8_t)clampi(g, 0, 255), bgr[2] = (uint8_t)clampi(r, 0, 255);
}

}  // namespace jpeg
}  // namespace ryolo
