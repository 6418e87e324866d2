// Baseline JPEG decode core, __host__ __device__ so that tests/native/jpeg_decode_host.cu runs the device's phases on
// the CPU (csrc/jpeg_decode.cu, deva/utils/jpeg_decode.py; the format rules are DESIGN §7).  The host has parsed the
// file, removed the stuffed 0x00 bytes and the RSTn markers from its scan, and cut every restart interval into
// subsequences; every function here is bounded by the ranges it is given and reports malformed data as a status.
//
// Entropy decode state: (bit position, block slot within the MCU, zig-zag index).  Two decodes that reach the same state
// agree from there on, which is what lets a subsequence be decoded from a guessed state and corrected later.
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif
#define JD_HD __host__ __device__ __forceinline__

namespace b200 {
namespace jpeg_decode {

enum Status {
  kOk = 0,
  kBadDescriptor = 1,
  kBadCode = 2,       // a code not in the table
  kBadCategory = 3,   // a DC category over 11 or an AC category over 10
  kRunPast63 = 4,     // a run or ZRL past coefficient 63
  kShortStream = 5,   // the interval's data ends before its last MCU
  kTrailing = 6,      // data left after the interval's last MCU
  kRange = 7,         // a block outside the range where libjpeg-turbo's C and x86 SIMD islow IDCTs agree
};

// Canonical Huffman lookup of one table: fast[top 9 bits] = length << 8 | symbol (0 for longer codes); a code of length
// l is `code <= maxcode[l]`, its symbol vals[code + valoff[l]].  int32 words, built by deva/utils/jpeg_decode.py.
constexpr int kFastBits = 9;
struct Huff {
  int32_t fast[1 << kFastBits];
  int32_t maxcode[18];
  int32_t valoff[18];
  int32_t vals[256];
};
// Per file: the DC and AC tables of each component and its quantisation table in natural order.
struct Tables {
  Huff huff[3][2];
  int32_t quant[3][64];
};
constexpr int kTableWords = (int)(sizeof(Tables) / 4);

// One file's descriptor: int64 [kDescFields] (include/deva_b200.h).
enum Field { kScanOff, kScanLen, kH, kW, kLumaH, kLumaV, kTablesIdx, kOutOff, kWorkOff, kFirstSub, kSubs, kDescFields };
// One restart interval: bits are positions in the batch's scan buffer, blocks count within the file.
enum IvField { kIvFile, kIvBitStart, kIvBitEnd, kIvFirstBlock, kIvBlocks, kIvFirstSub, kIvFields };
// One subsequence of an interval.
enum SubField { kSubInterval, kSubBitStart, kSubBitEnd, kSubFields };

constexpr int kMaxDim = 65535;

struct Geometry {
  int h, w, hy, vy, bpm, mcus_x, mcus_y;
  long long blocks;
  int plane_w[3], plane_h[3];
  JD_HD long long plane_bytes(int c) const { return (long long)plane_w[c] * plane_h[c]; }
};

// Y sampled hy x vy in {1x1, 2x1, 2x2}, Cb and Cr 1x1.
JD_HD bool geometry_of(long long h, long long w, long long hy, long long vy, Geometry* g) {
  if (h < 1 || w < 1 || h > kMaxDim || w > kMaxDim || !((hy == 1 && vy == 1) || (hy == 2 && vy == 1) ||
                                                          (hy == 2 && vy == 2)))
    return false;
  g->h = (int)h, g->w = (int)w, g->hy = (int)hy, g->vy = (int)vy, g->bpm = (int)(hy * vy + 2);
  g->mcus_x = (int)((w + 8 * hy - 1) / (8 * hy)), g->mcus_y = (int)((h + 8 * vy - 1) / (8 * vy));
  g->blocks = (long long)g->mcus_x * g->mcus_y * g->bpm;
  g->plane_w[0] = g->mcus_x * 8 * (int)hy, g->plane_h[0] = g->mcus_y * 8 * (int)vy;
  for (int c = 1; c < 3; ++c) g->plane_w[c] = g->mcus_x * 8, g->plane_h[c] = g->mcus_y * 8;
  return true;
}

JD_HD int component_of(const Geometry& g, int slot) {
  const int ny = g.hy * g.vy;
  return slot < ny ? 0 : slot - ny + 1;
}

// The state packed in one integer: bit position << 12 | slot << 7 | zig-zag index; kInvalid once a decode failed.
constexpr unsigned long long kInvalid = ~0ull;
JD_HD unsigned long long pack(long long pos, int slot, int zz) {
  return (unsigned long long)pos << 12 | (unsigned long long)slot << 7 | (unsigned long long)zz;
}
JD_HD long long pos_of(unsigned long long s) { return (long long)(s >> 12); }
JD_HD int slot_of(unsigned long long s) { return (int)(s >> 7) & 31; }
JD_HD int zz_of(unsigned long long s) { return (int)s & 127; }

// 32 bits from bit pos; bits at or past `end` (a byte boundary) read as ones.
JD_HD uint32_t peek32(const uint8_t* buf, long long end, long long pos) {
  const long long byte = pos >> 3;
  uint64_t v = 0;
  for (int k = 0; k < 5; ++k) v = v << 8 | ((byte + k) * 8 < end ? buf[byte + k] : 0xffu);
  return (uint32_t)(v >> (8 - (pos & 7)));
}

JD_HD int extend(uint32_t bits, int s) {
  return s == 0 ? 0 : (int)bits < (1 << (s - 1)) ? (int)bits - (1 << s) + 1 : (int)bits;
}

// The symbol at the top of `look` in table t: returns its length (0 when no code matches) and sets *sym.
JD_HD int huff_decode(const Huff& t, uint32_t look, int* sym) {
  const int f = t.fast[look >> (32 - kFastBits)];
  if (f) {
    *sym = f & 0xff;
    return f >> 8;
  }
  for (int l = kFastBits + 1; l <= 16; ++l) {
    const int code = (int)(look >> (32 - l));
    if (code <= t.maxcode[l]) {
      const int i = code + t.valoff[l];
      if (i < 0 || i > 255) return 0;
      *sym = t.vals[i];
      return l;
    }
  }
  return 0;
}

#ifdef __CUDA_ARCH__
__constant__
#endif
static const uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Decodes symbols from state *st while its bit position is below `stop` and fewer than `max_blocks` blocks have been
// completed.  Sink receives dc(component, difference), ac(natural index, value) and block_done().  Strict: a malformed
// symbol ends the decode with its Status and *st = kInvalid.  Lenient (the synchronisation phase, which decodes from
// guessed states): a code not in the table skips one bit, any category is read, and a run past coefficient 63 ends the
// block, so that a decode from a wrong guess keeps going until it falls into step with the true one.  On a valid stream
// the two agree.
template <bool kStrict, class Sink>
JD_HD int run(const Tables& t, const Geometry& g, const uint8_t* buf, long long end, long long stop,
              long long max_blocks, unsigned long long* st, Sink& sink) {
  if (*st == kInvalid) return kBadCode;
  long long pos = pos_of(*st);
  int slot = slot_of(*st), zz = zz_of(*st);
  long long done = 0;
  int status = kOk;
  while (pos < stop && done < max_blocks) {
    const uint32_t look = peek32(buf, end, pos);
    const int comp = component_of(g, slot);
    int sym;
    const int len = huff_decode(t.huff[comp][zz ? 1 : 0], look, &sym);
    if (!len) {
      if (kStrict) {
        status = kBadCode;
        break;
      }
      ++pos;
      continue;
    }
    const int s = sym & 15, r = sym >> 4;
    const uint32_t extra = s ? (look << len) >> (32 - s) : 0u;
    pos += len + s;
    bool complete = false;
    if (zz == 0) {
      if (kStrict && sym > 11) {
        status = kBadCategory;
        break;
      }
      sink.dc(comp, extend(extra, s));
      zz = 1;
    } else if (s) {
      if (kStrict && s > 10) {
        status = kBadCategory;
        break;
      }
      zz += r;
      if (zz > 63) {
        if (kStrict) {
          status = kRunPast63;
          break;
        }
        complete = true;
      } else {
        sink.ac(kNatural[zz], extend(extra, s));
        complete = ++zz == 64;
      }
    } else if (r == 15) {
      zz += 16;
      if (kStrict && zz > 64) {
        status = kRunPast63;
        break;
      }
      complete = zz >= 64;
    } else {
      complete = true;  // EOB
    }
    if (complete) {
      sink.block_done();
      zz = 0;
      if (++slot == g.bpm) slot = 0;
      ++done;
    }
  }
  *st = status == kOk ? pack(pos, slot, zz) : kInvalid;
  return status;
}

// What the synchronisation phase keeps of a decode: its exit state, completed blocks and per-component DC sums.
struct Exit {
  unsigned long long state;
  long long count;
  long long dc[3];
};

struct CountSink {
  long long count = 0, sums[3] = {0, 0, 0};
  JD_HD void dc(int c, int v) { sums[c] += v; }
  JD_HD void ac(int, int) {}
  JD_HD void block_done() { ++count; }
};

// Decode of one subsequence [start, stop) from state `entry` to the first symbol boundary at or past stop.
JD_HD Exit decode_sub(const Tables& t, const Geometry& g, const uint8_t* buf, long long end, long long stop,
                      unsigned long long entry) {
  CountSink sink;
  unsigned long long st = entry;
  run<false>(t, g, buf, end, stop, (long long)1 << 62, &st, sink);
  return Exit{st, sink.count, {sink.sums[0], sink.sums[1], sink.sums[2]}};
}

// The final pass's sink: writes int16 coefficients (natural order) into the file's blocks, starting at block `at`
// within [at, limit); DC values run from the predictors as libjpeg keeps them (int, stored as JCOEF).
struct WriteSink {
  int16_t* coef;
  long long at, limit;
  int pred[3];
  bool overflow = false;
  JD_HD void dc(int c, int v) {
    pred[c] += v;
    if (at < limit) coef[at * 64] = (int16_t)pred[c];
    else overflow = true;
  }
  JD_HD void ac(int k, int v) {
    if (at < limit) coef[at * 64 + k] = (int16_t)v;
    else overflow = true;
  }
  JD_HD void block_done() { ++at; }
};

// Position of a block (index in MCU order) in its component plane.
JD_HD void block_place(const Geometry& g, long long b, int* comp, int* bx, int* by) {
  const long long mcu = b / g.bpm;
  const int slot = (int)(b - mcu * g.bpm);
  const int mx = (int)(mcu % g.mcus_x), my = (int)(mcu / g.mcus_x);
  *comp = component_of(g, slot);
  if (*comp == 0) {
    *bx = mx * g.hy + slot % g.hy, *by = my * g.vy + slot / g.hy;
  } else {
    *bx = mx, *by = my;
  }
}

// jidctint.c's islow IDCT of one block (coef natural order, quant natural order) into 8x8 samples at out with row pitch
// `pitch`.  Returns kRange when the block leaves the range where libjpeg-turbo's C and x86 SIMD paths agree: a
// dequantised coefficient or a pass-1 output outside [-16383, 16383] (the SIMD code adds pairs of them in 16 bits), or
// an output before the range limit outside [-512, 511] (where range_limit[x & 1023] is not a clamp).
constexpr int kCoefLimit = 16383;
JD_HD int idct_islow(const int16_t* coef, const int32_t* quant, uint8_t* out, long long pitch) {
  constexpr int kConstBits = 13, kPass1Bits = 2;
  constexpr long long F0_298 = 2446, F0_390 = 3196, F0_541 = 4433, F0_765 = 6270, F0_899 = 7373, F1_175 = 9633,
                      F1_501 = 12299, F1_847 = 15137, F1_961 = 16069, F2_053 = 16819, F2_562 = 20995, F3_072 = 25172;
  int ws[64];
  bool bad = false;
  for (int c = 0; c < 8; ++c) {
    long long in[8];
    for (int r = 0; r < 8; ++r) {
      in[r] = (long long)coef[r * 8 + c] * quant[r * 8 + c];
      bad |= in[r] > kCoefLimit || in[r] < -kCoefLimit;
    }
    long long z2 = in[2], z3 = in[6];
    long long z1 = (z2 + z3) * F0_541;
    long long tmp2 = z1 + z3 * (-F1_847);
    long long tmp3 = z1 + z2 * F0_765;
    z2 = in[0], z3 = in[4];
    long long tmp0 = (z2 + z3) << kConstBits;
    long long tmp1 = (z2 - z3) << kConstBits;
    long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = in[7], tmp1 = in[5], tmp2 = in[3], tmp3 = in[1];
    z1 = tmp0 + tmp3, z2 = tmp1 + tmp2, z3 = tmp0 + tmp2;
    long long z4 = tmp1 + tmp3;
    long long z5 = (z3 + z4) * F1_175;
    tmp0 *= F0_298, tmp1 *= F2_053, tmp2 *= F3_072, tmp3 *= F1_501;
    z1 *= -F0_899, z2 *= -F2_562, z3 *= -F1_961, z4 *= -F0_390;
    z3 += z5, z4 += z5;
    tmp0 += z1 + z3, tmp1 += z2 + z4, tmp2 += z2 + z3, tmp3 += z1 + z4;
    const int sh = kConstBits - kPass1Bits;
    const long long rnd = 1ll << (sh - 1);
    long long o[8] = {(tmp10 + tmp3 + rnd) >> sh, (tmp11 + tmp2 + rnd) >> sh, (tmp12 + tmp1 + rnd) >> sh,
                      (tmp13 + tmp0 + rnd) >> sh, (tmp13 - tmp0 + rnd) >> sh, (tmp12 - tmp1 + rnd) >> sh,
                      (tmp11 - tmp2 + rnd) >> sh, (tmp10 - tmp3 + rnd) >> sh};
    for (int r = 0; r < 8; ++r) {
      bad |= o[r] > kCoefLimit || o[r] < -kCoefLimit;
      ws[r * 8 + c] = (int)o[r];
    }
  }
  for (int r = 0; r < 8; ++r) {
    const int* w = ws + r * 8;
    long long z2 = w[2], z3 = w[6];
    long long z1 = (z2 + z3) * F0_541;
    long long tmp2 = z1 + z3 * (-F1_847);
    long long tmp3 = z1 + z2 * F0_765;
    z2 = (long long)w[0] + (1ll << (kPass1Bits + 2));
    z3 = w[4];
    long long tmp0 = (z2 + z3) << kConstBits;
    long long tmp1 = (z2 - z3) << kConstBits;
    long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = w[7], tmp1 = w[5], tmp2 = w[3], tmp3 = w[1];
    z1 = tmp0 + tmp3, z2 = tmp1 + tmp2, z3 = tmp0 + tmp2;
    long long z4 = tmp1 + tmp3;
    long long z5 = (z3 + z4) * F1_175;
    tmp0 *= F0_298, tmp1 *= F2_053, tmp2 *= F3_072, tmp3 *= F1_501;
    z1 *= -F0_899, z2 *= -F2_562, z3 *= -F1_961, z4 *= -F0_390;
    z3 += z5, z4 += z5;
    tmp0 += z1 + z3, tmp1 += z2 + z4, tmp2 += z2 + z3, tmp3 += z1 + z4;
    const int sh = kConstBits + kPass1Bits + 3;
    long long o[8] = {(tmp10 + tmp3) >> sh, (tmp11 + tmp2) >> sh, (tmp12 + tmp1) >> sh, (tmp13 + tmp0) >> sh,
                      (tmp13 - tmp0) >> sh, (tmp12 - tmp1) >> sh, (tmp11 - tmp2) >> sh, (tmp10 - tmp3) >> sh};
    for (int c = 0; c < 8; ++c) {
      const long long v = o[c];
      bad |= v > 511 || v < -512;
      out[r * pitch + c] = (uint8_t)(v < -128 ? 0 : v > 127 ? 255 : v + 128);
    }
  }
  return bad ? kRange : kOk;
}

// One output pixel: Y from plane 0, Cb and Cr upsampled as libjpeg-turbo's h2v1 / h2v2 fancy upsampling (plain
// replication when the chroma width is at most 2), then jdcolor.c's fixed-point YCbCr -> RGB.
JD_HD int chroma_at(const Geometry& g, const uint8_t* p, int pw, int x, int y) {
  if (g.hy == 1) return p[(long long)y * pw + x];
  const int dw = (g.w + 1) / 2, dh = g.vy == 2 ? (g.h + 1) / 2 : g.h;
  const int i = x >> 1;
  if (dw <= 2) return p[(long long)(g.vy == 2 ? y >> 1 : y) * pw + i];
  const int ni = x & 1 ? (i + 1 < dw ? i + 1 : i) : (i > 0 ? i - 1 : 0);
  if (g.vy == 1) {
    const uint8_t* row = p + (long long)y * pw;
    return (3 * row[i] + row[ni] + (x & 1 ? 2 : 1)) >> 2;
  }
  const int j = y >> 1;
  const int nj = y & 1 ? (j + 1 < dh ? j + 1 : j) : (j > 0 ? j - 1 : 0);
  const uint8_t* r0 = p + (long long)j * pw;
  const uint8_t* r1 = p + (long long)nj * pw;
  const int c0 = 3 * r0[i] + r1[i], c1 = 3 * r0[ni] + r1[ni];
  return (3 * c0 + c1 + (x & 1 ? 7 : 8)) >> 4;
}

JD_HD uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }

JD_HD void ycc_to_rgb(int y, int cb, int cr, uint8_t* rgb) {
  constexpr int kScale = 16, kHalf = 1 << 15;
  const int xcb = cb - 128, xcr = cr - 128;
  const int r = (int)((91881ll * xcr + kHalf) >> kScale);
  const int b = (int)((116130ll * xcb + kHalf) >> kScale);
  const int gg = (int)((-46802ll * xcr + (-22554ll * xcb + kHalf)) >> kScale);
  rgb[0] = clamp255(y + r), rgb[1] = clamp255(y + gg), rgb[2] = clamp255(y + b);
}

}  // namespace jpeg_decode
}  // namespace b200
