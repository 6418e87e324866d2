// Baseline JPEG scan on the device: the entropy-coded segment (and EOI) of one RGB uint8 image, byte for byte what
// libjpeg(-turbo) writes for Pillow's default save at the given quantisation tables (DESIGN §7,
// deva/utils/jpeg_encode.py, oracle/jpeg_encode.py).  Every step is libjpeg's integer arithmetic, so the work is
// parallel over 8x8 blocks and the bytes are a function of the image and the tables alone:
//   1. blocks_kernel: 64 threads per MCU convert its 16x16 pixels to YCbCr (edge replication as libjpeg pads), 4:2:0
//      downsample, run the islow DCT and quantise; they write the six blocks' int16 zigzag coefficients in scan order
//      (dummy blocks past the image's last block column / row as libjpeg makes them);
//   2. huffman_kernel<false>: one warp per block counts its Huffman bits (the DC difference needs only the previous
//      block of the same component, already written);
//   3. scan_bits_kernel: one block scans the counts into bit offsets and ORs in the 1-bit fill;
//   4. huffman_kernel<true>: the same walk writes each lane's codes at its bit offset with atomicOr on a zeroed buffer;
//   5. stuffing: per 4 KiB segment count the 0xFF bytes, scan the counts, copy with a 0x00 after each 0xFF, append EOI.
#include <algorithm>
#include <stdint.h>

#include "common.h"
#include "scan.cuh"

namespace b200 {
namespace jpeg {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kMcusPerCta = 4;
constexpr int kWarps = 8;            // blocks per CTA of the Huffman kernels
constexpr int kScanThreads = 1024;
constexpr int kScanItems = 8;        // consecutive counts per scan thread
constexpr int kSegThreads = 256;
constexpr int kSegBytes = kSegThreads * 16;
constexpr int kMaxBlockBytes = 208;  // DC <= 22 bits + 63 AC codes <= 26 bits each, before stuffing

struct Tables {
  uint8_t q[2][64];  // luma, chroma quantisation tables, zigzag order
};

// ---- Annex K.3 Huffman tables, expanded at compile time to per-symbol codes --------------------------------------------
struct HuffSpec {
  uint8_t counts[16];
  uint8_t symbols[162];
};
struct HuffCodes {
  uint16_t code[256];
  uint8_t len[256];
};

constexpr HuffCodes derive(const HuffSpec& s) {
  HuffCodes t{};
  int code = 0, k = 0;
  for (int n = 1; n <= 16; ++n) {
    for (int c = 0; c < s.counts[n - 1]; ++c, ++k, ++code) {
      t.code[s.symbols[k]] = (uint16_t)code;
      t.len[s.symbols[k]] = (uint8_t)n;
    }
    code <<= 1;
  }
  return t;
}

constexpr HuffSpec kDcLuma{{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}};
constexpr HuffSpec kDcChroma{{0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}};
constexpr HuffSpec kAcLuma{
    {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
     0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
     0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
     0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
     0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
     0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
     0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
     0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
     0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};
constexpr HuffSpec kAcChroma{
    {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
     0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
     0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
     0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
     0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
     0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
     0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
     0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
     0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

__constant__ HuffCodes kDc[2] = {derive(kDcLuma), derive(kDcChroma)};
__constant__ HuffCodes kAc[2] = {derive(kAcLuma), derive(kAcChroma)};

// kZigzag[k]: natural (row-major) index of the k-th coefficient in zigzag order
__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ---- 1. colour, downsampling, DCT, quantisation ------------------------------------------------------------------------
__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// One pass of jfdctint.c's islow DCT over 8 values at stride s (rows, then columns with kLast).  Every intermediate
// fits int32: libjpeg's own C path uses 32-bit arithmetic for 8-bit samples.
template <bool kLast>
__device__ __forceinline__ void fdct_pass(int* d, int s) {
  constexpr int kConst = 13, kPass1 = 2, kShift = kLast ? kConst + kPass1 : kConst - kPass1;
  const int t0 = d[0] + d[7 * s], t7 = d[0] - d[7 * s];
  const int t1 = d[s] + d[6 * s], t6 = d[s] - d[6 * s];
  const int t2 = d[2 * s] + d[5 * s], t5 = d[2 * s] - d[5 * s];
  const int t3 = d[3 * s] + d[4 * s], t4 = d[3 * s] - d[4 * s];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  d[0] = kLast ? descale(t10 + t11, kPass1) : (t10 + t11) * (1 << kPass1);
  d[4 * s] = kLast ? descale(t10 - t11, kPass1) : (t10 - t11) * (1 << kPass1);
  const int z = (t12 + t13) * 4433;
  d[2 * s] = descale(z + t13 * 6270, kShift);
  d[6 * s] = descale(z - t12 * 15137, kShift);
  const int z5 = (t4 + t6 + t5 + t7) * 9633;
  const int z1 = (t4 + t7) * -7373, z2 = (t5 + t6) * -20995;
  const int z3 = (t4 + t6) * -16069 + z5, z4 = (t5 + t7) * -3196 + z5;
  d[7 * s] = descale(t4 * 2446 + z1 + z3, kShift);
  d[5 * s] = descale(t5 * 16819 + z2 + z4, kShift);
  d[3 * s] = descale(t6 * 25172 + z2 + z3, kShift);
  d[s] = descale(t7 * 12299 + z1 + z4, kShift);
}

// jccolor.c with FIX(x) = x * 2^16 rounded
__device__ __forceinline__ int luma(int r, int g, int b) { return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16; }
__device__ __forceinline__ int chroma_b(int r, int g, int b) {
  return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
}
__device__ __forceinline__ int chroma_r(int r, int g, int b) {
  return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

__global__ void __launch_bounds__(64 * kMcusPerCta) blocks_kernel(const uint8_t* __restrict__ img, int h, int w,
                                                                  int mcu_cols, int mcus, Tables tables,
                                                                  int16_t* __restrict__ coef) {
  __shared__ int sm[kMcusPerCta][6][64 + 1];  // +1: the row pass strides by 8 words
  const int g = threadIdx.x >> 6, t = threadIdx.x & 63;
  const int mcu = blockIdx.x * kMcusPerCta + g;
  const bool live = mcu < mcus;
  int(*blk)[65] = sm[g];
  const int my = mcu / mcu_cols, mx = mcu - my * mcu_cols;
  if (live) {
    // luma: row t / 4 of the MCU, 4 columns; the image's last row and column are replicated
    const int ly = t >> 2, y = min(my * 16 + ly, h - 1);
    for (int i = 0; i < 4; ++i) {
      const int lx = (t & 3) * 4 + i, x = min(mx * 16 + lx, w - 1);
      const uint8_t* p = img + ((long long)y * w + x) * 3;
      blk[(ly >> 3) * 2 + (lx >> 3)][(ly & 7) * 8 + (lx & 7)] = luma(__ldg(p), __ldg(p + 1), __ldg(p + 2)) - 128;
    }
    // chroma sample (t / 8, t % 8): rows past the downsampled plane's last repeat it; an odd last input row pairs
    // with itself
    const int cy = min(my * 8 + (t >> 3), (h + 1) / 2 - 1), cx = mx * 8 + (t & 7);
    int cb = 0, cr = 0;
    for (int dy = 0; dy < 2; ++dy)
      for (int dx = 0; dx < 2; ++dx) {
        const int y2 = min(2 * cy + dy, h - 1), x2 = min(2 * cx + dx, w - 1);
        const uint8_t* p = img + ((long long)y2 * w + x2) * 3;
        const int r = __ldg(p), gg = __ldg(p + 1), b = __ldg(p + 2);
        cb += chroma_b(r, gg, b);
        cr += chroma_r(r, gg, b);
      }
    const int bias = 1 + (cx & 1);
    blk[4][t] = ((cb + bias) >> 2) - 128;
    blk[5][t] = ((cr + bias) >> 2) - 128;
  }
  __syncthreads();
  if (live && t < 48) fdct_pass<false>(&blk[t >> 3][(t & 7) * 8], 1);
  __syncthreads();
  if (live && t < 48) fdct_pass<true>(&blk[t >> 3][t & 7], 8);
  __syncthreads();
  if (!live) return;
  // thread t quantises zigzag coefficient t of all six blocks
  const int nat = kZigzag[t];
  int v[6];
#pragma unroll
  for (int b = 0; b < 6; ++b) {
    const int c = blk[b][nat], d = 8 * tables.q[b >= 4][t];
    const int q = (abs(c) + (d >> 1)) / d;
    v[b] = c < 0 ? -q : q;
  }
  // dummy blocks: zero AC; the DC of the block to the left, or for a dummy block row of the MCU's upper-right block
  if (mx == mcu_cols - 1 && (((w + 7) >> 3) & 1)) {
    v[1] = t == 0 ? v[0] : 0;
    v[3] = t == 0 ? v[2] : 0;
  }
  if (my == (h + 15) / 16 - 1 && (((h + 7) >> 3) & 1)) v[2] = v[3] = t == 0 ? v[1] : 0;
  int16_t* out = coef + (long long)mcu * 6 * 64 + t;
#pragma unroll
  for (int b = 0; b < 6; ++b) out[b * 64] = (int16_t)v[b];
}

// ---- 2, 4. Huffman codes ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int magnitude_bits(int v) { return 32 - __clz(abs(v)); }

// n <= 27 bits of v (MSB first) at bit pos of a zeroed big-endian bit buffer
__device__ __forceinline__ void put_bits(uint32_t* words, unsigned long long pos, uint32_t v, int n) {
  const int s = (int)(pos & 31);
  const uint64_t x = (uint64_t)v << (64 - s - n);
  uint32_t* p = words + (pos >> 5);
  atomicOr(p, __byte_perm((uint32_t)(x >> 32), 0, 0x0123));
  if ((uint32_t)x) atomicOr(p + 1, __byte_perm((uint32_t)x, 0, 0x0123));
}

// One warp per block, lane l holding zigzag coefficients l and l + 32.  The tokens of coefficient k (its ZRLs, its run /
// size code and magnitude; the DC difference for k = 0) take bits[k]; EOB follows unless coefficient 63 is nonzero.
template <bool kEmit>
__global__ void __launch_bounds__(32 * kWarps) huffman_kernel(const int16_t* __restrict__ coef, long long blocks,
                                                              uint32_t* __restrict__ block_bits,
                                                              const unsigned long long* __restrict__ block_off,
                                                              uint32_t* __restrict__ words) {
  const int lane = threadIdx.x & 31;
  const long long b = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (b >= blocks) return;  // whole warps leave
  const int j = (int)(b % 6), tab = j >= 4;
  const int16_t* c = coef + b * 64;
  const int a = c[lane], z = c[lane + 32];
  const unsigned lo = __ballot_sync(kFull, a != 0) & ~1u, hi = __ballot_sync(kFull, z != 0);
  const uint64_t nz = lo | ((uint64_t)hi << 32);
  const HuffCodes& ac = kAc[tab];

  // slot 0: coefficient lane (the DC difference on lane 0); slot 1: coefficient lane + 32
  uint32_t code[2] = {0, 0};
  int len[2] = {0, 0}, zrl[2] = {0, 0};
  for (int slot = 0; slot < 2; ++slot) {
    const int k = lane + 32 * slot, v = slot ? z : a;
    if (k == 0) {
      long long prev = -1;  // the previous block of the component in scan order
      if (j == 0) prev = b - 3;
      else if (j < 4) prev = b - 1;
      else prev = b - 6;
      const int diff = v - (prev >= 0 ? coef[prev * 64] : 0), n = magnitude_bits(diff);
      const HuffCodes& dc = kDc[tab];
      code[0] = ((uint32_t)dc.code[n] << n) | ((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1));
      len[0] = dc.len[n] + n;
    } else if (v != 0) {
      const uint64_t below = nz & ((1ull << k) - 1);
      const int run = k - (below ? 63 - __clzll(below) : 0) - 1, n = magnitude_bits(v);
      const int sym = ((run & 15) << 4) | n;
      code[slot] = ((uint32_t)ac.code[sym] << n) | ((uint32_t)(v < 0 ? v - 1 : v) & ((1u << n) - 1));
      len[slot] = ac.len[sym] + n;
      zrl[slot] = run >> 4;
    }
  }
  const int zrl_len = ac.len[0xf0];
  const int bits0 = len[0] + zrl[0] * zrl_len, bits1 = len[1] + zrl[1] * zrl_len;
  int inc0 = bits0, inc1 = bits1;  // inclusive scans over the lanes
  for (int m = 1; m < 32; m <<= 1) {
    const int u0 = __shfl_up_sync(kFull, inc0, m), u1 = __shfl_up_sync(kFull, inc1, m);
    if (lane >= m) inc0 += u0, inc1 += u1;
  }
  const int total0 = __shfl_sync(kFull, inc0, 31), total1 = __shfl_sync(kFull, inc1, 31);
  const bool eob = !(nz >> 63);
  if (!kEmit) {
    if (lane == 0) block_bits[b] = (uint32_t)(total0 + total1 + (eob ? ac.len[0] : 0));
    return;
  }
  const unsigned long long base = block_off[b];
  unsigned long long pos[2] = {base + inc0 - bits0, base + total0 + inc1 - bits1};
  for (int slot = 0; slot < 2; ++slot) {
    for (int r = 0; r < zrl[slot]; ++r, pos[slot] += zrl_len) put_bits(words, pos[slot], ac.code[0xf0], zrl_len);
    if (len[slot]) put_bits(words, pos[slot], code[slot], len[slot]);
  }
  if (eob && lane == 0) put_bits(words, base + total0 + total1, ac.code[0], ac.len[0]);
}

// ---- 3, 5. scans --------------------------------------------------------------------------------------------------------
// Exclusive scan of n counts into off, kScanItems consecutive counts per thread; returns the total on every thread.
__device__ unsigned long long scan_counts(const uint32_t* __restrict__ counts, long long n,
                                          unsigned long long* __restrict__ off) {
  __shared__ unsigned long long warp_sums[kScanThreads / 32];
  return block_scan<kScanItems>(
      n, 0ull, warp_sums, [&](long long i) { return counts[i]; },
      [&](long long i, unsigned long long o, uint32_t) { off[i] = o; });
}

// The 0xFF bytes among the 16 of q
__device__ __forceinline__ int count_ff(const uint4& q) {
  return (__popc(__vcmpeq4(q.x, kFull)) + __popc(__vcmpeq4(q.y, kFull)) + __popc(__vcmpeq4(q.z, kFull)) +
          __popc(__vcmpeq4(q.w, kFull))) >> 3;
}

// meta[0]: bytes of the scan before stuffing; the fill's 1-bits are ORed into its last byte.
__global__ void __launch_bounds__(kScanThreads) scan_bits_kernel(const uint32_t* __restrict__ block_bits,
                                                                 long long blocks,
                                                                 unsigned long long* __restrict__ block_off,
                                                                 uint32_t* __restrict__ words,
                                                                 unsigned long long* __restrict__ meta) {
  const unsigned long long bits = scan_counts(block_bits, blocks, block_off);
  if (threadIdx.x != 0) return;
  const int fill = (int)(-(long long)bits & 7);
  if (fill) put_bits(words, bits, (1u << fill) - 1, fill);
  meta[0] = (bits + 7) >> 3;
}

// 16 bytes per thread, kSegBytes per block: the segment's 0xFF count
__global__ void __launch_bounds__(kSegThreads) count_ff_kernel(const uint4* __restrict__ bytes,
                                                               const unsigned long long* __restrict__ meta,
                                                               uint32_t* __restrict__ seg_ff) {
  __shared__ unsigned long long warp_sums[kSegThreads / 32];
  const unsigned long long n = meta[0];
  if ((unsigned long long)blockIdx.x * kSegBytes >= n) return;  // past the scan: whole blocks leave
  const uint4 q = bytes[(long long)blockIdx.x * kSegThreads + threadIdx.x];  // bytes past n are zero
  unsigned long long total;
  block_exclusive_scan<unsigned long long>(count_ff(q), warp_sums, total);
  if (threadIdx.x == 0) seg_ff[blockIdx.x] = (uint32_t)total;
}

// The segments' output offsets (before their own bytes), EOI and the stuffed length.
__global__ void __launch_bounds__(kScanThreads) scan_ff_kernel(const uint32_t* __restrict__ seg_ff,
                                                               unsigned long long* __restrict__ seg_off,
                                                               const unsigned long long* __restrict__ meta,
                                                               uint8_t* __restrict__ out, int64_t* __restrict__ out_len) {
  const unsigned long long n = meta[0];
  const unsigned long long ff = scan_counts(seg_ff, (long long)((n + kSegBytes - 1) / kSegBytes), seg_off);
  if (threadIdx.x != 0) return;
  out[n + ff] = 0xff;
  out[n + ff + 1] = 0xd9;
  *out_len = (int64_t)(n + ff + 2);
}

__global__ void __launch_bounds__(kSegThreads) stuff_kernel(const uint4* __restrict__ bytes,
                                                            const unsigned long long* __restrict__ meta,
                                                            const unsigned long long* __restrict__ seg_off,
                                                            uint8_t* __restrict__ out) {
  __shared__ unsigned long long warp_sums[kSegThreads / 32];
  const unsigned long long n = meta[0];
  if ((unsigned long long)blockIdx.x * kSegBytes >= n) return;
  const uint4 q = bytes[(long long)blockIdx.x * kSegThreads + threadIdx.x];
  unsigned long long total;
  const unsigned long long before = block_exclusive_scan<unsigned long long>(count_ff(q), warp_sums, total);
  const unsigned long long p0 = (unsigned long long)blockIdx.x * kSegBytes + threadIdx.x * 16;
  uint8_t* dst = out + p0 + seg_off[blockIdx.x] + before;
  const uint32_t word[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    if (p0 + i >= n) break;
    const uint8_t v = (uint8_t)(word[i >> 2] >> (8 * (i & 3)));
    *dst++ = v;
    if (v == 0xff) *dst++ = 0;
  }
}

// ---- sizes --------------------------------------------------------------------------------------------------------------
inline long long blocks_of(int h, int w) { return 6LL * ((h + 15) / 16) * ((w + 15) / 16); }
inline long long segments_of(int h, int w) { return (blocks_of(h, w) * kMaxBlockBytes + 1 + kSegBytes - 1) / kSegBytes; }
// Workspace regions, each 16-byte aligned.
struct Work {
  int16_t* coef;                  // [blocks * 64]
  uint32_t* block_bits;           // [blocks]
  unsigned long long* block_off;  // [blocks]
  uint32_t* seg_ff;               // [segments]
  unsigned long long* seg_off;    // [segments]
  unsigned long long* meta;       // [1]
  uint32_t* words;                // the scan before stuffing, segments * kSegBytes bytes
};

inline size_t carve(int h, int w, void* base, Work* wk) {
  const long long nb = blocks_of(h, w), ns = segments_of(h, w);
  Carver<16> c{static_cast<char*>(base)};
  Work t;
  t.coef = c.take<int16_t>(nb * 64);
  t.block_bits = c.take<uint32_t>(nb);
  t.block_off = c.take<unsigned long long>(nb);
  t.seg_ff = c.take<uint32_t>(ns);
  t.seg_off = c.take<unsigned long long>(ns);
  t.meta = c.take<unsigned long long>(1);
  t.words = c.take<uint32_t>(ns * (kSegBytes / 4));
  if (wk) *wk = t;
  return c.bytes;
}

}  // namespace jpeg
}  // namespace b200

using namespace b200;

extern "C" {

DEVA_B200_API size_t deva_b200_jpeg_bound(int h, int w) {
  return (size_t)(2 * (jpeg::blocks_of(h, w) * jpeg::kMaxBlockBytes + 1) + 2);
}

DEVA_B200_API size_t deva_b200_jpeg_workspace_bytes(int h, int w) { return jpeg::carve(h, w, nullptr, nullptr); }

DEVA_B200_API int deva_b200_jpeg_encode(const uint8_t* img, int h, int w, const uint8_t* quality_tables,
                                        void* workspace, uint8_t* out, int64_t* out_len, deva_stream_t stream) {
  B200_REQUIRE(img && quality_tables && workspace && out && out_len && h > 0 && w > 0 && h <= 65535 && w <= 65535,
               "jpeg_encode: bad arguments");
  B200_REQUIRE(((uintptr_t)workspace & 15) == 0, "jpeg_encode: workspace must be 16-byte aligned");
  jpeg::Tables tables;
  for (int i = 0; i < 128; ++i) {
    B200_REQUIRE(quality_tables[i] >= 1, "jpeg_encode: quantisation table entry %d is 0", i);
    tables.q[i / 64][i % 64] = quality_tables[i];
  }
  jpeg::Work ws;
  jpeg::carve(h, w, workspace, &ws);
  const int mcu_cols = (w + 15) / 16, mcus = ((h + 15) / 16) * mcu_cols;
  const long long blocks = jpeg::blocks_of(h, w), segs = jpeg::segments_of(h, w);
  cudaStream_t s = S(stream);
  B200_CUDA(cudaMemsetAsync(ws.words, 0, (size_t)segs * jpeg::kSegBytes, s));
  jpeg::blocks_kernel<<<ceil_div(mcus, jpeg::kMcusPerCta), 64 * jpeg::kMcusPerCta, 0, s>>>(img, h, w, mcu_cols, mcus,
                                                                                           tables, ws.coef);
  B200_LAUNCH_CHECK();
  const unsigned hb = (unsigned)ceil_div(blocks, jpeg::kWarps);
  jpeg::huffman_kernel<false><<<hb, 32 * jpeg::kWarps, 0, s>>>(ws.coef, blocks, ws.block_bits, nullptr, nullptr);
  B200_LAUNCH_CHECK();
  jpeg::scan_bits_kernel<<<1, jpeg::kScanThreads, 0, s>>>(ws.block_bits, blocks, ws.block_off, ws.words, ws.meta);
  B200_LAUNCH_CHECK();
  jpeg::huffman_kernel<true><<<hb, 32 * jpeg::kWarps, 0, s>>>(ws.coef, blocks, nullptr, ws.block_off, ws.words);
  B200_LAUNCH_CHECK();
  const uint4* bytes = reinterpret_cast<const uint4*>(ws.words);
  jpeg::count_ff_kernel<<<(unsigned)segs, jpeg::kSegThreads, 0, s>>>(bytes, ws.meta, ws.seg_ff);
  B200_LAUNCH_CHECK();
  jpeg::scan_ff_kernel<<<1, jpeg::kScanThreads, 0, s>>>(ws.seg_ff, ws.seg_off, ws.meta, out, out_len);
  B200_LAUNCH_CHECK();
  jpeg::stuff_kernel<<<(unsigned)segs, jpeg::kSegThreads, 0, s>>>(bytes, ws.meta, ws.seg_off, out);
  B200_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
