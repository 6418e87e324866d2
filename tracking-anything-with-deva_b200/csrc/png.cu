// PNG image data on the device: the zlib stream of one uint8 image in the fixed format of DESIGN §7
// (deva/utils/png_encode.py, oracle/png_encode.py).  Every row is Up-filtered on the fly from the source, tokenised on
// its own (greedy matches at distances 1 and bpp, fixed Huffman codes), so rows are independent and the work is
// parallel over rows:
//   1. rows_kernel<false>: one warp per row stages the row's filtered bytes (and the 4 before them) in shared memory,
//      walks its tokens and counts their bits; it also forms the row's Adler-32 partial sums;
//   2. frame_kernel: one block scans the bit counts into each row's bit offset, zeroes the words two rows share,
//      writes the zlib header, the block header, end-of-block, the Adler-32 trailer and the stream's length;
//   3. rows_kernel<true>: the same walk writes each row's bits at its offset.  Words inside a row are plain stores;
//      a row's first and last words may be shared with its neighbours and take atomicOr.  The output is deterministic.
// The walk is uniform across the warp: a match length is found 32 positions at a time with a ballot.
#include <algorithm>
#include <stdint.h>

#include "common.h"
#include "scan.cuh"

namespace b200 {
namespace png {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kLookback = 4;  // staged bytes before the row (distances are at most 3)
constexpr int kMaxMatch = 258;
constexpr int kMaxWarps = 8;
constexpr int kScanThreads = 1024;
constexpr uint32_t kAdlerMod = 65521;
constexpr long long kFirstRowBit = 16 + 3;  // after the zlib header (2 bytes) and the block header (BFINAL, BTYPE = 01)

__constant__ uint16_t kLenBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                      31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};

struct Shape {
  const uint8_t* img;
  int w, channels, bits;
  int seg;  // bytes of a row segment of the filtered stream: filter byte + packed row
  int bpp;  // bytes per complete pixel, at least 1
};

// Byte k of row y as Pillow packs it: 8-bit rows are the pixels' bytes; sub-byte rows pack MSB-first with zero padding,
// a pixel taking v & (2^bits - 1) at 2 and 4 bits and v != 0 at 1 bit.
__device__ __forceinline__ uint32_t raw_byte(const Shape& g, long long y, int k) {
  if (g.bits == 8) return __ldg(g.img + y * g.w * g.channels + k);
  const int ppb = 8 / g.bits;
  const uint8_t* row = g.img + y * g.w;
  uint32_t b = 0;
  for (int t = 0; t < ppb; ++t) {
    const int x = k * ppb + t;
    uint32_t v = x < g.w ? __ldg(row + x) : 0u;
    v = g.bits == 1 ? (v != 0) : v & ((1u << g.bits) - 1);
    b |= v << (8 - g.bits * (t + 1));
  }
  return b;
}

// Byte p of the filtered stream s.
__device__ __forceinline__ uint8_t stream_byte(const Shape& g, long long p) {
  const long long y = p / g.seg;
  const int i = (int)(p - y * g.seg);
  if (i == 0) return 2;
  const uint32_t prev = y > 0 ? raw_byte(g, y - 1, i - 1) : 0u;
  return (uint8_t)(raw_byte(g, y, i - 1) - prev);
}

// Run of s[j] == s[j - d] from row position i, at most `limit` long; sm[kLookback + i] is the row's byte i.
__device__ __forceinline__ int run_length(const uint8_t* sm, long long o, int i, int d, int limit, int lane) {
  if (o + i - d < 0) return 0;
  const uint8_t* a = sm + kLookback + i;
  for (int base = 0; base < limit; base += 32) {
    const int k = base + lane;
    const bool same = k < limit && a[k] == a[k - d];
    const unsigned differ = __ballot_sync(kFull, !same);
    if (differ) return base + __ffs(differ) - 1;
  }
  return limit;
}

__device__ __forceinline__ uint32_t reverse_bits(uint32_t code, int n) { return __brev(code) >> (32 - n); }

// Bits written at a bit offset of a word buffer (LSB-first, as deflate orders them).  The row's first word and its
// trailing partial word may be shared with the neighbouring rows: atomicOr on words the frame kernel zeroed.
struct BitWriter {
  uint32_t* out;
  long long word;
  uint64_t acc;
  int n;
  bool first;
  bool lane0;

  __device__ void put(uint32_t v, int bits) {
    acc |= (uint64_t)v << n;
    n += bits;
    if (n >= 32) {
      if (lane0) {
        if (first) atomicOr(out + word, (uint32_t)acc);
        else out[word] = (uint32_t)acc;
      }
      acc >>= 32;
      n -= 32;
      ++word;
      first = false;
    }
  }
  __device__ void finish() {
    if (n > 0 && lane0) atomicOr(out + word, (uint32_t)acc);
  }
};

template <bool kEmit>
__device__ __forceinline__ void literal(BitWriter& bw, uint64_t& bits, uint32_t v) {
  const int n = v <= 143 ? 8 : 9;
  if (kEmit) bw.put(reverse_bits(v <= 143 ? 0x30 + v : 0x190 + v - 144, n), n);
  else bits += n;
}

template <bool kEmit>
__device__ __forceinline__ void match(BitWriter& bw, uint64_t& bits, int len, int d) {
  int k = 28;
  if (len < kMaxMatch) {
    k = 27;
    while (kLenBase[k] > len) --k;
  }
  const int sym = 257 + k, n = sym <= 279 ? 7 : 8;
  const int extra = kLenExtra[k];
  if (kEmit) {
    bw.put(reverse_bits(sym <= 279 ? sym - 256 : 0xC0 + sym - 280, n), n);
    if (extra) bw.put(len - kLenBase[k], extra);
    bw.put(reverse_bits(d - 1, 5), 5);  // distance codes 0..3 are distances 1..4, no extra bits
  } else {
    bits += n + extra + 5;
  }
}

// One warp per row.  Counting pass: row_bits, row_sum (sum of the row's bytes) and row_weighted (sum of (seg - k) * s_k,
// mod 65521).  Emitting pass: the row's tokens at row_off.
template <bool kEmit>
__global__ void __launch_bounds__(32 * kMaxWarps) rows_kernel(Shape g, int h, int stride, uint32_t* __restrict__ row_bits,
                                                            uint32_t* __restrict__ row_sum,
                                                            uint32_t* __restrict__ row_weighted,
                                                            const unsigned long long* __restrict__ row_off,
                                                            uint32_t* __restrict__ out) {
  extern __shared__ uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long y = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
  if (y >= h) return;  // whole warps leave
  uint8_t* sm = smem + (size_t)warp * stride;
  const int seg = g.seg;
  const long long o = y * seg;
  for (int t = lane; t < seg + kLookback; t += 32) {
    const long long p = o - kLookback + t;
    if (p >= 0) sm[t] = stream_byte(g, p);
  }
  __syncwarp();

  if (!kEmit) {
    uint64_t sum = 0, weighted = 0;
    for (int k = lane; k < seg; k += 32) {
      const uint32_t v = sm[kLookback + k];
      sum += v;
      weighted += (uint64_t)(seg - k) * v;
    }
    for (int m = 16; m; m >>= 1) {
      sum += __shfl_xor_sync(kFull, sum, m);
      weighted += __shfl_xor_sync(kFull, weighted, m);
    }
    if (lane == 0) {
      row_sum[y] = (uint32_t)sum;
      row_weighted[y] = (uint32_t)(weighted % kAdlerMod);
    }
  }

  BitWriter bw{out, 0, 0, 0, true, lane == 0};
  if (kEmit) {
    const unsigned long long b = row_off[y];
    bw.word = (long long)(b >> 5);
    bw.n = (int)(b & 31);
  }
  uint64_t bits = 0;
  for (int i = 0; i < seg;) {
    const int limit = min(seg - i, kMaxMatch);
    int best = run_length(sm, o, i, 1, limit, lane), dist = 1;
    if (g.bpp > 1) {
      const int r = run_length(sm, o, i, g.bpp, limit, lane);
      if (r > best) best = r, dist = g.bpp;
    }
    if (best >= 3) {
      match<kEmit>(bw, bits, best, dist);
      i += best;
    } else {
      literal<kEmit>(bw, bits, sm[kLookback + i]);
      i += 1;
    }
  }
  if (kEmit) bw.finish();
  else if (lane == 0) row_bits[y] = (uint32_t)bits;
}

// One block: bit offsets of the rows, the stream's framing and its length.
__global__ void __launch_bounds__(kScanThreads) frame_kernel(int h, int seg, const uint32_t* __restrict__ row_bits,
                                                             const uint32_t* __restrict__ row_sum,
                                                             const uint32_t* __restrict__ row_weighted,
                                                             unsigned long long* __restrict__ row_off,
                                                             uint32_t* __restrict__ out, int64_t* __restrict__ out_len) {
  __shared__ unsigned long long warp_sums[kScanThreads / 32];
  __shared__ unsigned long long s1_total, s2_total;
  const int tid = threadIdx.x;
  const long long n = (long long)h * seg;
  if (tid == 0) s1_total = s2_total = 0;
  unsigned long long s1 = 0, s2 = 0;
  // end_bit follows the last row; end-of-block is seven 0 bits
  const unsigned long long end_bit = block_scan(
      h, (unsigned long long)kFirstRowBit, warp_sums, [&](long long r) { return row_bits[r]; },
      [&](long long r, unsigned long long off, uint32_t v) {
        row_off[r] = off;
        out[off >> 5] = 0;  // the row's first and last words, shared with the neighbouring rows
        out[(off + v - 1) >> 5] = 0;
        const long long after = n - r * seg - seg;  // bytes of s after the row
        s1 += row_sum[r];
        s2 += row_weighted[r] + (unsigned long long)(after % kAdlerMod) * (row_sum[r] % kAdlerMod) % kAdlerMod;
      });
  atomicAdd(&s1_total, s1);
  atomicAdd(&s2_total, s2);
  __syncthreads();
  if (tid != 0) return;
  // s1 = 1 + sum s_k; s2 = sum over k of the running s1 = n + sum (n - k) s_k
  const uint32_t a = (uint32_t)((1 + s1_total) % kAdlerMod);
  const uint32_t b = (uint32_t)((n % kAdlerMod + s2_total) % kAdlerMod);
  out[0] |= 0x78u | (0x01u << 8) | (3u << 16);  // zlib CMF, FLG; then BFINAL = 1, BTYPE = 01
  const long long body = (long long)((end_bit + 7 + 7) >> 3);
  uint8_t* bytes = reinterpret_cast<uint8_t*>(out);
  for (long long k = (long long)((end_bit + 7) >> 3); k < body; ++k) bytes[k] = 0;
  const uint32_t adler = (b << 16) | a;
  for (int k = 0; k < 4; ++k) bytes[body + k] = (uint8_t)(adler >> (24 - 8 * k));
  *out_len = body + 4;
}

inline long long stream_bytes(int h, int w, int channels, int bits) {
  return (long long)h * (((long long)w * channels * bits + 7) / 8 + 1);
}

// Workspace regions, each 8-byte aligned.
struct Work {
  uint32_t* row_stats;          // [3 * h] row_bits, row_sum, row_weighted
  unsigned long long* row_off;  // [h]
};

inline size_t carve(int h, void* base, Work* wk) {
  Carver<8> c{static_cast<char*>(base)};
  Work t;
  t.row_stats = c.take<uint32_t>(3ll * h);
  t.row_off = c.take<unsigned long long>(h);
  if (wk) *wk = t;
  return c.bytes;
}

}  // namespace png
}  // namespace b200

using namespace b200;

extern "C" {

DEVA_B200_API size_t deva_b200_png_bound(int h, int w, int channels, int bits) {
  const long long n = png::stream_bytes(h, w, channels, bits);
  const long long bound = (3 + 9 * n + 7 + 7) / 8 + 6;
  return (size_t)((bound + 3) / 4 * 4);
}

DEVA_B200_API size_t deva_b200_png_workspace_bytes(int h) { return png::carve(h, nullptr, nullptr); }

DEVA_B200_API int deva_b200_png_encode(const uint8_t* img, int h, int w, int channels, int bits, void* workspace,
                                       uint8_t* out, int64_t* out_len, deva_stream_t stream) {
  B200_REQUIRE(img && workspace && out && out_len && h > 0 && w > 0, "png_encode: bad arguments");
  B200_REQUIRE((channels == 1 && (bits == 1 || bits == 2 || bits == 4 || bits == 8)) || (channels == 3 && bits == 8),
               "png_encode: %d channels at %d bits, expected 1 channel at 1, 2, 4 or 8 bits or 3 at 8", channels, bits);
  B200_REQUIRE(((uintptr_t)out & 3) == 0 && ((uintptr_t)workspace & 7) == 0,
               "png_encode: out must be 4-byte and workspace 8-byte aligned");
  const long long seg = ((long long)w * channels * bits + 7) / 8 + 1;
  const int stride = (int)((seg + png::kLookback + 15) / 16 * 16);
  int max_smem = 0;
  B200_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, device_slot()));
  B200_REQUIRE(stride <= max_smem, "png_encode: a row of %lld bytes does not fit in shared memory", seg - 1);
  const int warps = (int)std::max(1, std::min(png::kMaxWarps, 48 * 1024 / stride));
  const size_t smem = (size_t)warps * stride;
  png::Shape g{img, w, channels, bits, (int)seg, std::max(1, channels * bits / 8)};
  png::Work wk;
  png::carve(h, workspace, &wk);
  uint32_t* row_bits = wk.row_stats;
  uint32_t* row_sum = row_bits + h;
  uint32_t* row_weighted = row_sum + h;
  unsigned long long* row_off = wk.row_off;
  uint32_t* words = reinterpret_cast<uint32_t*>(out);
  cudaStream_t s = S(stream);
  const unsigned blocks = (unsigned)ceil_div(h, warps);
  if (smem > 48 * 1024) {
    B200_CUDA(cudaFuncSetAttribute(png::rows_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    B200_CUDA(cudaFuncSetAttribute(png::rows_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  png::rows_kernel<false><<<blocks, 32 * warps, smem, s>>>(g, h, stride, row_bits, row_sum, row_weighted, nullptr,
                                                           nullptr);
  B200_LAUNCH_CHECK();
  png::frame_kernel<<<1, png::kScanThreads, 0, s>>>(h, (int)seg, row_bits, row_sum, row_weighted, row_off, words,
                                                    out_len);
  B200_LAUNCH_CHECK();
  png::rows_kernel<true><<<blocks, 32 * warps, smem, s>>>(g, h, stride, nullptr, nullptr, nullptr, row_off, words);
  B200_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
