// Inflate of one zlib stream (RFC 1950 framing around RFC 1951 deflate) into a buffer of known length: the core of
// png_decode.cu, written once for the device and the host so that a CPU build of the same code can be tested against
// zlib (tests/test_png_decode_cpu.py builds tests/native/inflate_host.cu).
//
// A stream is accepted (status kOk) only when it is one well-formed zlib stream: a valid header without a preset
// dictionary; blocks that zlib's inflate would accept (stored LEN == ~NLEN; code-length sets neither over-subscribed
// nor incomplete, except a literal/length or distance code of a single 1-bit code; no literal/length symbol 286/287,
// no distance code 30/31, no distance before the stream's start); exactly `out_len` inflated bytes, ending with the
// final block; the Adler-32 trailer right after it, matching; and no byte after the trailer.  Every read of the input
// is bounded by its length and every write by out_len, so a malformed stream ends in a status, never out of bounds.
//
// One thread decodes the symbols (Inflater::run).  It writes literals and short matches itself and hands every match
// of at least `min_copy` bytes back to its caller as a pending copy, which the device's warp performs in parallel:
// out[at + j] = out[at - dist + j % dist] reads only bytes before `at`, so the lanes need no order among themselves.
// Matches read their source from `win`, the last kWindow bytes of the output (shared memory on the device), never from
// `out` itself.  kWindow exceeds deflate's largest distance plus its longest match, so a copy's reads never alias its
// writes in the window.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define INFLATE_HD __host__ __device__ __forceinline__
#else
#define INFLATE_HD inline
#endif

namespace b200 {
namespace inflate {

enum Status : int {
  kOk = 0,
  kBadHeader = 1,       // CMF / FLG: method 8, window <= 32 KiB, check bits, no preset dictionary
  kBadBlockType = 2,    // BTYPE 3
  kBadStored = 3,       // LEN != ~NLEN
  kBadCodeLengths = 4,  // over-subscribed or incomplete code, a repeat without a length or past the end, no end-of-block
  kBadSymbol = 5,       // an unused code, literal/length symbol 286/287 or distance code 30/31
  kBadDistance = 6,     // a distance before the stream's start
  kTooLong = 7,         // more than out_len inflated bytes
  kTruncated = 8,       // the input ends inside the stream
  kTooShort = 9,        // the final block ends before out_len bytes
  kBadAdler = 10,       // the trailer does not match the inflated bytes
  kTrailing = 11,       // bytes after the trailer
  kBadFilter = 12,      // (png_decode.cu) a row's filter type is over 4
  kBadDescriptor = 13,  // (png_decode.cu) a descriptor outside the supported shapes and formats
  kCopyPending = -1,    // run() returns to let its caller perform a long match copy
};

constexpr uint32_t kAdlerMod = 65521;
constexpr int kFastBits = 10;  // codes of at most this many bits decode with one table lookup
constexpr int kWindow = 1 << 16;  // > 32768 + 258
constexpr long long kWindowMask = kWindow - 1;

// Little-endian bit reader over in[0, len); bytes past the end read as zero and make overrun() true once consumed.
struct Bits {
  const uint8_t* in;
  long long len;
  long long next;  // next byte to load into buf
  uint64_t buf;
  int cnt;  // bits in buf

  INFLATE_HD void refill() {
    while (cnt <= 56) {
      buf |= (uint64_t)(next < len ? in[next] : 0) << cnt;
      ++next;
      cnt += 8;
    }
  }
  INFLATE_HD uint32_t peek(int n) {  // n <= 32
    refill();
    return (uint32_t)(buf & ((1ull << n) - 1));
  }
  INFLATE_HD void drop(int n) {
    buf >>= n;
    cnt -= n;
  }
  INFLATE_HD uint32_t get(int n) {
    const uint32_t v = peek(n);
    drop(n);
    return v;
  }
  INFLATE_HD long long consumed_bits() const { return next * 8 - cnt; }
  INFLATE_HD bool overrun() const { return consumed_bits() > len * 8; }
};

// A canonical Huffman code (RFC 1951 §3.2.2): fast[] maps the next kFastBits input bits to (symbol << 4 | length) for
// codes of at most kFastBits bits (0 elsewhere); longer codes are found by walking count[] and sym[].
struct Huff {
  uint16_t fast[1 << kFastBits];
  uint16_t count[16];  // codes of each length
  uint16_t sym[288];   // symbols ordered by (length, value): the order of their codes
};

struct Tables {
  Huff lit, dist;
  uint8_t lens[288 + 32];
};

INFLATE_HD uint32_t reverse_bits(uint32_t v, int n) {
  uint32_t r = 0;
  for (int i = 0; i < n; ++i) r |= ((v >> i) & 1u) << (n - 1 - i);
  return r;
}

// Builds the code of symbols 0..n-1 with code lengths lens[] (0: unused).  A set with no code at all is accepted (any
// use of it fails); an incomplete set is refused, except a literal/length or distance code of a single 1-bit code
// (lengths_code false), which zlib accepts.
INFLATE_HD int build(Huff& h, const uint8_t* lens, int n, bool lengths_code) {
  for (int l = 0; l < 16; ++l) h.count[l] = 0;
  for (int s = 0; s < n; ++s) h.count[lens[s]]++;
  h.count[0] = 0;
  int left = 1, max_len = 0;
  for (int l = 1; l < 16; ++l) {
    left = 2 * left - h.count[l];
    if (left < 0) return kBadCodeLengths;  // over-subscribed
    if (h.count[l]) max_len = l;
  }
  if (max_len > 0 && left > 0 && (lengths_code || max_len != 1)) return kBadCodeLengths;  // incomplete
  uint16_t offs[16];
  offs[1] = 0;
  for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + h.count[l];
  for (int s = 0; s < n; ++s)
    if (lens[s]) h.sym[offs[lens[s]]++] = (uint16_t)s;
  for (int i = 0; i < (1 << kFastBits); ++i) h.fast[i] = 0;
  uint32_t code = 0;
  int k = 0;
  for (int l = 1; l <= kFastBits; ++l) {  // the codes of one length are consecutive; the next length starts at 2x
    for (int c = 0; c < h.count[l]; ++c, ++k, ++code) {
      const uint16_t e = (uint16_t)(h.sym[k] << 4 | l);
      for (uint32_t i = reverse_bits(code, l); i < (1u << kFastBits); i += 1u << l) h.fast[i] = e;
    }
    code <<= 1;
  }
  return kOk;
}

// The next symbol of code h, or -1 for a code the set does not use.
INFLATE_HD int decode(Bits& b, const Huff& h) {
  const uint32_t e = h.fast[b.peek(kFastBits)];
  if (e) {
    b.drop(e & 15);
    return (int)(e >> 4);
  }
  const uint32_t bits = b.peek(15);
  int code = 0, first = 0, index = 0;
  for (int l = 1; l < 16; ++l) {
    code |= (bits >> (l - 1)) & 1;
    const int c = h.count[l];
    if (code >= first && code - first < c) {
      b.drop(l);
      return h.sym[index + code - first];
    }
    index += c;
    first = (first + c) << 1;
    code <<= 1;
  }
  return -1;
}

// Length and distance symbols (RFC 1951 §3.2.5): base values and extra bits, from their regular structure.
INFLATE_HD int length_extra(int k) { return k < 8 || k == 28 ? 0 : (k - 4) >> 2; }  // k = symbol - 257
INFLATE_HD int length_base(int k) {
  return k < 8 ? 3 + k : k == 28 ? 258 : ((4 + ((k - 4) & 3)) << length_extra(k)) + 3;
}
INFLATE_HD int dist_extra(int d) { return d < 4 ? 0 : (d - 2) >> 1; }
INFLATE_HD int dist_base(int d) { return d < 4 ? d + 1 : ((2 + (d & 1)) << dist_extra(d)) + 1; }

// The code lengths of a dynamic block (after BFINAL and BTYPE) into t, then its two codes.
INFLATE_HD int read_dynamic(Bits& b, Tables& t) {
  const int hlit = (int)b.get(5) + 257, hdist = (int)b.get(5) + 1, hclen = (int)b.get(4) + 4;
  if (hlit > 286 || hdist > 30) return kBadCodeLengths;
  const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  uint8_t cl[19];
  for (int i = 0; i < 19; ++i) cl[order[i]] = i < hclen ? (uint8_t)b.get(3) : 0;
  int st = build(t.lit, cl, 19, true);
  if (st) return st;
  const int total = hlit + hdist;
  for (int i = 0; i < total;) {
    if (b.overrun()) return kTruncated;
    const int sym = decode(b, t.lit);
    if (sym < 0) return kBadCodeLengths;
    if (sym < 16) {
      t.lens[i++] = (uint8_t)sym;
      continue;
    }
    int rep;
    uint8_t v = 0;
    if (sym == 16) {
      if (i == 0) return kBadCodeLengths;
      v = t.lens[i - 1];
      rep = 3 + (int)b.get(2);
    } else if (sym == 17) {
      rep = 3 + (int)b.get(3);
    } else {
      rep = 11 + (int)b.get(7);
    }
    if (i + rep > total) return kBadCodeLengths;
    while (rep--) t.lens[i++] = v;
  }
  if (b.overrun()) return kTruncated;
  if (t.lens[256] == 0) return kBadCodeLengths;  // no end-of-block
  st = build(t.lit, t.lens, hlit, false);
  if (st) return st;
  return build(t.dist, t.lens + hlit, hdist, false);
}

INFLATE_HD int read_fixed(Tables& t) {
  for (int s = 0; s < 288; ++s) t.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
  int st = build(t.lit, t.lens, 288, false);
  if (st) return st;
  for (int s = 0; s < 32; ++s) t.lens[s] = 5;
  return build(t.dist, t.lens, 32, false);
}

struct Inflater {
  enum Phase { kZlibHeader, kBlockHeader, kCodes, kStored, kTrailer, kDone };
  Bits bits;
  uint8_t* out;
  uint8_t* win;  // kWindow bytes: out[p] is also win[p & kWindowMask]
  long long out_len, pos;
  int phase, final_block;
  long long stored_left;
  long long copy_at;  // a pending copy: out[copy_at + j] = out[copy_at - copy_dist + j % copy_dist], j < copy_len
  int copy_len, copy_dist;
  uint32_t adler;  // the trailer's value, once read

  INFLATE_HD void init(const uint8_t* in, long long in_len, uint8_t* dst, long long dst_len, uint8_t* window) {
    bits = Bits{in, in_len, 0, 0, 0};
    out = dst;
    win = window;
    out_len = dst_len;
    pos = 0;
    phase = kZlibHeader;
    final_block = 0;
    stored_left = 0;
    copy_at = 0;
    copy_len = copy_dist = 0;
    adler = 0;
  }

  INFLATE_HD void put(long long p, uint8_t v) {
    out[p] = v;
    win[p & kWindowMask] = v;
  }
  // The source byte of position at + j of a match at distance dist.
  INFLATE_HD uint8_t source(long long at, int dist, int j) const { return win[(at - dist + j % dist) & kWindowMask]; }

  // Decodes until the stream's trailer has been read (kOk: the caller checks `adler`), a match of at least min_copy
  // bytes is pending (kCopyPending; pos already counts it), or the stream is refused (a positive status).
  INFLATE_HD int run(Tables& t, int min_copy) {
    Bits& b = bits;
    for (;;) {
      if (b.overrun()) return kTruncated;
      switch (phase) {
        case kZlibHeader: {
          const uint32_t cmf = b.get(8), flg = b.get(8);
          if ((cmf & 15) != 8 || (cmf >> 4) > 7 || (cmf * 256 + flg) % 31 != 0 || (flg & 32)) return kBadHeader;
          phase = kBlockHeader;
          break;
        }
        case kBlockHeader: {
          if (final_block) {
            if (pos != out_len) return kTooShort;
            phase = kTrailer;
            break;
          }
          final_block = (int)b.get(1);
          const uint32_t type = b.get(2);
          int st = kOk;
          if (type == 0) {
            b.drop(b.cnt & 7);  // to the byte boundary
            const uint32_t len = b.get(16), nlen = b.get(16);
            if (len != (~nlen & 0xffffu)) return kBadStored;
            if ((long long)len > out_len - pos) return kTooLong;
            stored_left = len;
            phase = kStored;
            break;
          }
          if (type == 1) st = read_fixed(t);
          else if (type == 2) st = read_dynamic(b, t);
          else return kBadBlockType;
          if (st) return st;
          phase = kCodes;
          break;
        }
        case kStored: {
          while (stored_left > 0) {
            if (b.overrun()) return kTruncated;
            put(pos++, (uint8_t)b.get(8));
            --stored_left;
          }
          phase = kBlockHeader;
          break;
        }
        case kCodes: {
          for (;;) {
            if (b.overrun()) return kTruncated;
            const int sym = decode(b, t.lit);
            if (sym < 0 || sym > 285) return kBadSymbol;
            if (sym < 256) {
              if (pos >= out_len) return kTooLong;
              put(pos++, (uint8_t)sym);
              continue;
            }
            if (sym == 256) break;
            const int k = sym - 257;
            const int len = length_base(k) + (int)b.get(length_extra(k));
            const int d = decode(b, t.dist);
            if (d < 0 || d > 29) return kBadSymbol;
            const int dist = dist_base(d) + (int)b.get(dist_extra(d));
            if (dist > pos) return kBadDistance;
            if (len > out_len - pos) return kTooLong;
            if (len >= min_copy) {
              copy_at = pos;
              copy_len = len;
              copy_dist = dist;
              pos += len;
              return kCopyPending;
            }
            for (int j = 0; j < len; ++j) put(pos + j, win[(pos - dist + j) & kWindowMask]);
            pos += len;
          }
          phase = kBlockHeader;
          break;
        }
        case kTrailer: {
          b.drop(b.cnt & 7);
          uint32_t a = 0;
          for (int i = 0; i < 4; ++i) a = a << 8 | b.get(8);
          adler = a;
          if (b.overrun()) return kTruncated;
          if (b.consumed_bits() != b.len * 8) return kTrailing;
          phase = kDone;
          return kOk;
        }
        default:
          return kOk;
      }
    }
  }
};

// Adler-32 of bytes[0, n), serially (the device forms it from per-lane partial sums).
INFLATE_HD uint32_t adler32(const uint8_t* bytes, long long n) {
  uint32_t a = 1, b = 0;
  for (long long i = 0; i < n; ++i) {
    a = (a + bytes[i]) % kAdlerMod;
    b = (b + a) % kAdlerMod;
  }
  return b << 16 | a;
}

}  // namespace inflate
}  // namespace b200
