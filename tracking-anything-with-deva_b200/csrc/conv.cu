// Implicit-GEMM convolution on wgmma, NHWC fp16 activations, fp32 accumulation in registers.
// Replaces the nn.Conv2d + BatchNorm(eval) + ReLU (+ residual add) call chains of the reference network
// (deva/model/resnet.py:46-152, big_modules.py:23-212, modules.py:22-169, group_modules.py:41-67).
//
//   D[pixel, cout] = sum_{tap, cin} X[b, y*s + dy(tap), x*s + dx(tap), cin] * W[cout, tap, cin]
//
//   M = 128 output pixels = a TH x TW rectangle of one image, or (flat tiles, stride 1) 128 consecutive pixels of one
//   image in row-major order; N = NT output channels (<= 256), K = 64 input channels of one filter tap per k-iteration.
//
// A operand: the activation tensor is described to TMA as a rank-5 tiled tensor (C, W, H, B, 1); the box
//   (64, TW, TH, 1, 1) lands in shared memory as 128 rows of 128 bytes in exactly the 128B-swizzled K-major
//   layout wgmma wants.  A filter tap is just a shifted box origin; convolution padding is TMA's
//   out-of-bounds zero fill (also for negative coordinates).  Stride-2 convolutions use one tensor map per
//   input phase (y%2, x%2) over the same memory, so every tap is again a unit-stride box.
//   Flat tiles: no rectangle of 128 pixels fits an output like 68 x 120, and the best one, (1, 128), spends 6.25 % of
//   the MMA rows on padding.  A flat tile t of image b is pixels 128t .. 128t+127 of that image, loaded through an
//   im2col-mode tensor map (rank 4: C, W, H, B): the load starts at the tile's first output pixel shifted by -pad, walks
//   128 pixels through the bounding box of filter-window origins, and a filter tap is the im2col offset (dx, dy) + pad.
//   Padding is again the zero fill.  Rows past the image's last pixel read the next image (or the zero fill) and
//   compute values that are never stored; the staged epilogue's maps see the image as [B, 1, Ho*Wo, C].
// B operand: weights packed [Cout_pad, taps * Cin_pad] fp16 (K-major), 2-D TMA.
// Epilogue (straight from the accumulator registers): + bias (folded BatchNorm), + optional residual (own or
//   batch-broadcast), + optional rank-1 term w1[cout] * x1[b, pixel] (the "+1" mask / logit input channel of
//   sensory_compress and g4_conv), then writes any of: raw fp16, ReLU'd fp16, raw fp32.
//   Staged form (full-width tiles, at most three 8/16-bit outputs): after a tile's k-iterations the producer fills
//   N/64 more ring stages, one per 64-channel chunk, with the chunk's residual box (hi in the A slot, lo in the B slot)
//   or, without a residual, reserves them.  The consumers read the residual from the stage, write their outputs into
//   it in place and one thread drains them with TMA stores, which clip at the image edge.  Otherwise (ragged Cout,
//   split-K fp32 partials, the gate epilogue, larger output sets) residuals are loaded and outputs stored per thread.
//   After the k-loop the kernel runs epilogue_staged, epilogue_regs (per thread) or epilogue_gates.  The first two share
//   the pair arithmetic (pair_value, pair_store), the head (head_weights, head_add, head_store) and the row -> pixel
//   map (tile_row, row_pixel), so that they produce identical bits.  Odd Cout (per thread only) has its own
//   element-wise finish_scalar.
// Warp roles: warps 0..7 = two consumer warpgroups (pixels 0..63 / 64..127 of the tile: wgmma m64nNk16 + epilogue),
//   warps 8..11 = producer warpgroup, of which one thread issues the TMA loads.  The producer warpgroup exists so
//   that setmaxnreg can hand its registers to the consumers (a 64 x 256 fp32 accumulator is 128 registers per
//   thread).  Persistent CTAs, 4-stage shared-memory ring; the producer fills the ring for the next tile while the
//   consumers run the epilogue of the current one.
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include <type_traits>

#include "common.h"
#include "ptx.cuh"
#include "tmap.h"

namespace b200 {
namespace conv {

constexpr int BM = 128, BK = 64;
constexpr int STAGES = 4;
constexpr int A_BYTES = BM * BK * 2;
constexpr int B_BYTES_MAX = 256 * BK * 2;
constexpr int STAGE_BYTES = A_BYTES + B_BYTES_MAX;
constexpr int RING_BYTES = STAGES * STAGE_BYTES;
constexpr int CONSUMER_THREADS = 256;  // two warpgroups; wgmma needs warpgroups aligned to warp 0, 4, ...
constexpr int THREADS = CONSUMER_THREADS + 128;
// Per-thread registers after setmaxnreg.  The launch gives every thread 65536 / 384 -> 168; the producer warpgroup
// returns 128 each, which is exactly the 64 more each consumer takes.
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
static_assert(128 * PRODUCER_REGS + CONSUMER_THREADS * CONSUMER_REGS <= THREADS * 168, "conv: register budget");
constexpr int kMaxTaps = 32;  // k-entries (filter tap x pass) of one launch
constexpr int kMaxHead = 9;   // outputs of the fused 1x1 head
// Head weights in shared memory, per column pair (c, c + 1): the 9 taps' (w[t][c], w[t][c + 1]) side by side, padded to
// 20 floats so that a pair's weights are 4 x 16 B + 8 B loads and the four pairs a quad reads at once (80 B apart) hit
// disjoint banks.
constexpr int kHeadPairStride = 20;
constexpr int HEAD_BYTES = 128 * kHeadPairStride * 4;
constexpr int kMaxBias = 2048;   // bias of the whole layer staged in shared memory (Cout_pad <= kMaxBias)
constexpr int kMaxRank1 = 1024;  // same for the rank-1 input column
constexpr int SMEM_BYTES = RING_BYTES + 256 + HEAD_BYTES + kMaxBias * 4 + kMaxRank1 * 4;
static_assert(SMEM_BYTES <= 232448, "conv: shared-memory budget");

struct Params {
  int batch, ho, wo, cout;
  int tiles_x, tiles_y, tw, th;
  // flat tiles (flat_wo = the output width > 0): everything but the activation loads sees each output image as one row,
  // ho = 1, wo = Ho * Wo, tiled by th x tw = 1 x 128; the loads recover the pixel's (y, x) from flat_wo.  pad: the
  // filter's padding (a tap's im2col offset is its input offset + pad).
  int flat_wo, pad;
  int n_tiles, nt;
  int taps, cblocks;
  int m_tiles;   // batch * tiles_y * tiles_x
  int units;     // m_tiles * n_tiles * ksplit work units (read from the parameter bank: no register held across a tile)
  signed char tap_map[kMaxTaps], tap_w[kMaxTaps], tap_dx[kMaxTaps], tap_dy[kMaxTaps];  // per k-entry: activation
                                                         // map, weight tap group, input offset
  const float* bias;
  const __half* res;
  const __half* res_lo;
  long long res_batch_stride;  // elements; 0 = broadcast one image over the batch
  const float* rank1_w;
  const float* rank1_x;        // [batch, ho*wo]
  __half* out_raw;
  __half* out_relu;
  float* out_f32;
  __half* out_raw_lo;
  __half* out_relu_lo;
  const float* head_w;
  float* head_out;
  int head_n;
  const __half* gate_h;  // EPI_GATES: previous hidden state [batch, ho, wo, gate_c]
  __half* gate_out;
  int gate_c;
  // split-K (fp32 output only): unit = (k-split, tile); split ks accumulates k-iterations [ks*k_per_split, ...) in its own
  // accumulator and writes its partial sum to out_f32 + ks*f32_split_stride (bias in split 0).  The consumer adds
  // the partials in fp32 on the CUDA cores: the tensor core's accumulator rounds toward zero at every step, which
  // costs a split-precision conv with a deep K loop ~1e-5 relative (tools/accum_probe.py); short chains do not.
  int ksplit, k_per_split;
  long long f32_split_stride;
  // fp8 correction entries (split_mode 3): k-entries [0, taps16) are fp16 passes of `cblocks` 64-channel blocks, entries
  // [taps16, taps) are e4m3 x e4m3 passes of `cblocks8` 128-channel blocks over the 8-bit low-order activation tensor
  // and the 8-bit weights; both feed the same accumulator, which the epilogue scales by acc_scale.  The e4m3 k-iterations
  // run FIRST: wgmma adds e4m3 products to the accumulator with a reduced-precision adder (~14 significant bits of the
  // running sum), which is harmless relative to the small correction term alone but would drop most of it on top of the
  // full fp16 sum (~2e-4 relative error); the fp16 passes then accumulate on top in fp32.
  int taps16, cblocks8;
  float acc_scale;
  uint8_t* out_relu_lo8;  // optional: e4m3 of (relu - fp16(relu)) * 4096, the low-order operand of the next fp8 pass
  // staged epilogue: 1 = through the ring (see the file comment).  Each wanted output owns one 16 KB region of a stage:
  // region 0 = the A slot (where the residual's hi part lands), 1 / 2 = the halves of the B slot (lo part in 1).  fp16
  // regions hold the chunk as 128 rows of 128 B, 128B-swizzled like the residual box; the e4m3 region 64 B rows.
  int staged;
  __half* out_pool4;  // staged only: [batch, ho/4, wo/4, cout] 4x4 average of the raw output (raw staged, maybe not stored)
  int store_mask;                                          // bit k: region k is stored through maps.out[k]
  signed char reg_raw, reg_raw_lo, reg_relu, reg_relu_lo, reg_lo8;  // region of each output (when wanted)
};

struct Maps {
  CUtensorMap act[8];     // box {64, tw, th}; flat tiles: im2col, 128 pixels x 64 channels
  CUtensorMap wgt;        // box {64, nt}
  CUtensorMap act8;       // e4m3 low-order activations, box {128 B, tw, th}; flat tiles: im2col, 128 pixels x 128 B
  CUtensorMap wgt8;       // e4m3 weights, box {128 B, nt}
  CUtensorMap res, res_lo;  // staged epilogue: residual (hi, lo) [B or 1, Ho, Wo, Cout], box {64, tw, th}
  CUtensorMap out[3];       // staged epilogue: the output stored from region k, box {64, tw, th}
                            // (flat tiles: [B or 1, 1, Ho*Wo, Cout], box {64, 128, 1})
};

__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, const int (&c)[5]) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c[0]), "r"(c[1]), "r"(c[2]), "r"(c[3]), "r"(c[4])
      : "memory");
}

// Im2col load of 128 pixels (flat tiles): c = (channel, x, y, image) of the first pixel's filter-window origin,
// (dx, dy) the tap's offset inside the window.
__device__ __forceinline__ void tma_load_im2col_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, const int (&c)[4],
                                                   uint16_t dx, uint16_t dy) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c[0]), "r"(c[1]), "r"(c[2]), "r"(c[3]), "h"(dx), "h"(dy)
      : "memory");
}

// e4m3 pair {lo : low byte, hi : high byte}
__device__ __forceinline__ uint16_t to_e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
// (a - fp16(a)) * 4096 of a ReLU'd value a: the 8-bit low-order operand of an fp8 correction pass
__device__ __forceinline__ float lo8_value(float a) { return (a - __half2float(__float2half_rn(a))) * 4096.f; }

// Work unit `u` -> tile.  Units enumerate (k-split, channel tile, pixel tile).
__device__ __forceinline__ void tile_decode(int u, const Params& p, int& b, int& y0, int& x0, int& n0, int& ks) {
  ks = u % p.ksplit;
  u /= p.ksplit;
  const int nidx = u % p.n_tiles;
  int m = u / p.n_tiles;
  const int tx = m % p.tiles_x;
  m /= p.tiles_x;
  const int ty = m % p.tiles_y;
  b = m / p.tiles_y;
  y0 = ty * p.th;
  x0 = tx * p.tw;
  n0 = nidx * p.nt;
}

// EPI selects the epilogue: plain (bias / residual / rank-1 / ReLU / outputs), plain + fused logit head, or the gated
// hidden-state update of the sensory updaters.
enum { EPI_PLAIN = 0, EPI_HEAD = 1, EPI_GATES = 2 };

// Gate non-linearities of the fused hidden-state update.  ex2.approx + rcp.approx: absolute error < 1e-6 (the state is
// stored in fp16, 5e-4), ~6 instructions each instead of ~15 (IEEE division) / ~40 (tanhf with its branchy slow path).
// exp overflow -> +inf -> quotient 0 -> the correct limits 0 / 1 / -1.
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float tanh_fast(float x) { return 1.f - __fdividef(2.f, 1.f + __expf(2.f * x)); }

// One column pair (channels ch, ch + 1) of one row, in both plain / head forms.  The callers pass the pair's addresses:
// global per thread, the stage's regions staged.  Which terms and outputs apply is read from Params, not from null
// addresses: the compiler cannot prove a ring address non-null, and a null test per element splits the bias's
// multiply-add (other bits) and spills.  (v0, v1): the accumulator times acc_scale, scaled by the callers where every use
// of the product shares the block, which keeps that fusion as it was.  Then the bias (when add_bias), the rank-1 term
// w1[ch] * x1 and the residual's hi and lo parts; the terms stay conditional, as adding a zero turns -0 into +0.
__device__ __forceinline__ float2 pair_value(const Params& p, float v0, float v1, bool add_bias, const float* bias,
                                             const float* r1w, float r1x, const __half* res, const __half* res_lo) {
  if (add_bias) { v0 += bias[0]; v1 += bias[1]; }
  if (p.rank1_w) { v0 = fmaf(r1w[0], r1x, v0); v1 = fmaf(r1w[1], r1x, v1); }
  if (p.res) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(res));
    v0 += f.x; v1 += f.y;
  }
  if (p.res_lo) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(res_lo));
    v0 += f.x; v1 += f.y;
  }
  return make_float2(v0, v1);
}
// fp16 of (v0, v1) and, when `with_lo`, the fp16 of what that rounding dropped
__device__ __forceinline__ void store_hi_lo(__half* hi, bool with_lo, __half* lo, float v0, float v1) {
  const __half2 h = __floats2half2_rn(v0, v1);
  *reinterpret_cast<__half2*>(hi) = h;
  if (with_lo) {
    const float2 back = __half22float2(h);
    *reinterpret_cast<__half2*>(lo) = __floats2half2_rn(v0 - back.x, v1 - back.y);
  }
}
__device__ __forceinline__ float2 relu2(float2 v) { return make_float2(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f)); }
// The pair's raw fp16 (also for the 4x4 pool, staged) and ReLU'd fp16 outputs with their lo parts, and the e4m3
// operand of the next fp8 pass.  a = relu2(v), taken once by the caller for these and the head: a ReLU inside each
// branch was duplicated into both arms of the next (one more branch per pair in the staged head loop).
__device__ __forceinline__ void pair_store(const Params& p, float2 v, float2 a, __half* raw, __half* raw_lo, __half* relu,
                                           __half* relu_lo, uint8_t* lo8) {
  if (p.out_raw || p.out_pool4) store_hi_lo(raw, p.out_raw_lo, raw_lo, v.x, v.y);
  if (p.out_relu) store_hi_lo(relu, p.out_relu_lo, relu_lo, a.x, a.y);
  if (p.out_relu_lo8) *reinterpret_cast<uint16_t*>(lo8) = to_e4m3x2(lo8_value(a.x), lo8_value(a.y));
}

// One element of an odd Cout (unaligned pairs; per-thread form only): its own copy of the terms and conversions.  Its
// unconditional `ks == 0 ? bias : 0` (the sign of a zero on later k-splits) and its fusion are kept as they were.
// `e`: element offset of (pixel, channel) in the [pixels, cout] outputs; `rc` relative to the residual row.
__device__ __forceinline__ float finish_scalar(const Params& p, float o, int ch, long long e, const __half* res,
                                              const __half* res_lo, int rc, float r1x, int ks) {
  o += ks == 0 ? p.bias[ch] : 0.f;
  if (p.rank1_w) o = fmaf(p.rank1_w[ch], r1x, o);
  if (res) o += __half2float(res[rc]);
  if (res_lo) o += __half2float(res_lo[rc]);
  if (p.out_raw) {
    const __half hv = __float2half_rn(o);
    p.out_raw[e] = hv;
    if (p.out_raw_lo) p.out_raw_lo[e] = __float2half_rn(o - __half2float(hv));
  }
  if (p.out_relu) {
    const float ro = fmaxf(o, 0.f);
    const __half hv = __float2half_rn(ro);
    p.out_relu[e] = hv;
    if (p.out_relu_lo) p.out_relu_lo[e] = __float2half_rn(ro - __half2float(hv));
  }
  if (p.out_relu_lo8) p.out_relu_lo8[e] = (uint8_t)(to_e4m3x2(lo8_value(fmaxf(o, 0.f)), 0.f) & 0xffu);
  if (p.out_f32) p.out_f32[ks * p.f32_split_stride + e] = o;
  return o;
}

// Fused logit head (9 taps over the ReLU'd channels, fp32): w[2t + e] = tap t's weight of channel 8j + 2qd + e.
__device__ __forceinline__ void head_weights(const float* s_head, int j, int qd, float (&w)[2 * kMaxHead]) {
  const float* hw = s_head + (4 * j + qd) * kHeadPairStride;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 f = reinterpret_cast<const float4*>(hw)[q];
    w[4 * q] = f.x; w[4 * q + 1] = f.y; w[4 * q + 2] = f.z; w[4 * q + 3] = f.w;
  }
  const float2 f = reinterpret_cast<const float2*>(hw)[8];
  w[16] = f.x; w[17] = f.y;
}
// Adds a pair's ReLU'd values (a0, a1) to a pixel's running sums.  Both forms take the pairs in ascending order, a1
// before a0, so their sums agree bit for bit.
__device__ __forceinline__ void head_add(float (&acc)[kMaxHead], const float (&w)[2 * kMaxHead], float a0, float a1) {
#pragma unroll
  for (int t = 0; t < kMaxHead; ++t) acc[t] = fmaf(a0, w[2 * t], fmaf(a1, w[2 * t + 1], acc[t]));
}
// The four threads of a quad hold the same pixel's sums over disjoint channels: reduce them, and the quad's first thread
// stores the pixel's head_n outputs (pix < 0: past the image edge, nothing stored).
__device__ __forceinline__ void head_store(const Params& p, float (&acc)[kMaxHead], long long pix, int qd) {
#pragma unroll
  for (int t = 0; t < kMaxHead; ++t) {
    acc[t] += __shfl_xor_sync(0xffffffffu, acc[t], 1);
    acc[t] += __shfl_xor_sync(0xffffffffu, acc[t], 2);
  }
  if (pix >= 0 && qd == 0) {
#pragma unroll
    for (int t = 0; t < kMaxHead; ++t)
      if (t < p.head_n) p.head_out[pix * p.head_n + t] = acc[t];
  }
}

// Consumer thread (warp, lane) holds tile rows 16 warp + lane / 4 + 8i (i = 0, 1): wgmma's fragment layout.
__device__ __forceinline__ int tile_row(int warp, int lane, int i) { return 16 * warp + (lane >> 2) + 8 * i; }
// Tile row r of the tile at (b, y0, x0): its pixel index in [batch, ho, wo], or -1 past the image edge.
__device__ __forceinline__ long long row_pixel(const Params& p, int b, int y0, int x0, int r) {
  const int ty = r / p.tw, y = y0 + ty, x = x0 + r - ty * p.tw;
  return (y < p.ho && x < p.wo) ? ((long long)b * p.ho + y) * p.wo + x : -1ll;
}

// Shared memory: the ring's A and B slots and barriers, then the head weights, the bias and the rank-1 column.
struct Smem {
  uint8_t *sA, *sB;
  uint64_t *full, *empty;
  float *head, *bias, *r1w;  // [128 pairs][kHeadPairStride] head weights, [kMaxBias] bias, [kMaxRank1] rank-1 column
};

// Staged form (see the file comment): the tile's N / 64 chunks through the ring stages the producer issued after its
// k-iterations.  Rows past the image edge read the zero fill and compute values that no store writes.
template <int N, bool HEAD>
__device__ __forceinline__ void epilogue_staged(const Maps& maps, const Params& p, const Smem& s, const float (&d)[N / 2],
                                                int& stage, uint32_t& phase, int b, int y0, int x0, int n0) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, qd = lane & 3;
  // The rows' pixels are recomputed where used: only the accumulators, head sums and rank-1 inputs stay live.
  float r1x[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const long long pix = row_pixel(p, b, y0, x0, tile_row(warp, lane, i));
    r1x[i] = (p.rank1_x && pix >= 0) ? p.rank1_x[pix] : 0.f;
  }
  float hacc[2][HEAD ? kMaxHead : 1];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int t = 0; t < (HEAD ? kMaxHead : 1); ++t) hacc[i][t] = 0.f;
  int prev = 0;
#pragma unroll
  for (int c = 0; c < N / 64; ++c) {
    mbar_wait(&s.full[stage], phase);
    uint8_t* const slot_a = s.sA + stage * A_BYTES;
    uint8_t* const slot_b = s.sB + stage * B_BYTES_MAX;
    auto region = [&](const int k) { return k == 0 ? slot_a : slot_b + (k - 1) * A_BYTES; };
#pragma unroll
    for (int jl = 0; jl < 8; ++jl) {  // column block of the chunk; the thread reads and writes the same elements
      const int j = 8 * c + jl;
      float w[2 * kMaxHead];
      if constexpr (HEAD) head_weights(s.head, j, qd, w);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = tile_row(warp, lane, i);
        const uint32_t o16 = r * 128 + (((jl ^ (r & 7)) << 4) | (qd << 2));  // 128B swizzle: conflict-free
        const int ch = n0 + 8 * j + 2 * qd;
        auto at = [&](const int k) { return reinterpret_cast<__half*>(region(k) + o16); };
        const float2 v = pair_value(p, d[4 * j + 2 * i] * p.acc_scale, d[4 * j + 2 * i + 1] * p.acc_scale, true,
                                    s.bias + ch, s.r1w + ch, r1x[i], at(0), at(1));
        const float2 a = relu2(v);
        pair_store(p, v, a, at(p.reg_raw), at(p.reg_raw_lo), at(p.reg_relu), at(p.reg_relu_lo),
                   region(p.reg_lo8) + r * 64 + 8 * jl + 2 * qd);
        if constexpr (HEAD) head_add(hacc[i], w, a.x, a.y);
      }
    }
    fence_proxy_async();  // this thread's writes -> the TMA store's reads
    named_bar_sync(1, CONSUMER_THREADS);
    if (threadIdx.x == 0) {
      const int cc[5] = {n0 + 64 * c, x0, y0, b, 0};
      for (int k = 0; k < 3; ++k)
        if (p.store_mask >> k & 1) tma_store_5d(&maps.out[k], region(k), cc);
      bulk_commit();
      if (c > 0) {  // the previous chunk's stores have read their stage: hand it back to the producer
        bulk_wait_read<1>();
        mbar_arrive(&s.empty[prev], CONSUMER_THREADS);
      }
    }
    if (p.out_pool4) {
      // 4x4 windows of the staged raw chunk in area_down_kernel's order (fp32 sum from 0 over dy, then dx, then
      // * 1/16, one fp16 rounding), so the result is area_down(raw, 4) bit for bit.  The tile holds 8 windows;
      // warp w takes window w, lane l its channel pair 2l: one 128-byte row per read, conflict-free.
      const int win = warp, pc = lane;
      const int wy = win / (p.tw >> 2), wx = win - wy * (p.tw >> 2);
      const uint8_t* raw = region(p.reg_raw);
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int dy = 0; dy < 4; ++dy)
#pragma unroll
        for (int dx = 0; dx < 4; ++dx) {
          const int r = (4 * wy + dy) * p.tw + 4 * wx + dx;
          const float2 f = __half22float2(
              *reinterpret_cast<const __half2*>(raw + r * 128 + ((((pc >> 2) ^ (r & 7)) << 4) | ((pc & 3) << 2))));
          s0 += f.x; s1 += f.y;
        }
      const int y = y0 + 4 * wy, x = x0 + 4 * wx;
      if (y < p.ho && x < p.wo)  // ho, wo are multiples of 4: a window is wholly inside or wholly outside
        *reinterpret_cast<__half2*>(
            p.out_pool4 + (((long long)b * (p.ho >> 2) + (y >> 2)) * (p.wo >> 2) + (x >> 2)) * p.cout + n0 + 64 * c + 2 * pc) =
            __floats2half2_rn(s0 * 0.0625f, s1 * 0.0625f);
    }
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  if (p.out_pool4) named_bar_sync(1, CONSUMER_THREADS);  // every thread has read the last chunk for the pool
  if (threadIdx.x == 0) {
    bulk_wait_read<0>();
    mbar_arrive(&s.empty[prev], CONSUMER_THREADS);
  }
  if constexpr (HEAD) {
#pragma unroll
    for (int i = 0; i < 2; ++i) head_store(p, hacc[i], row_pixel(p, b, y0, x0, tile_row(warp, lane, i)), qd);
  }
}

// Per-thread form of the plain / head epilogue: residuals read and outputs written straight from the accumulator
// registers.  It takes every launch the staged form does not (ragged Cout, split-K fp32 partials, larger output sets).
template <int N, bool HEAD>
__device__ __forceinline__ void epilogue_regs(const Params& p, const Smem& s, const float (&d)[N / 2], int b, int y0,
                                              int x0, int n0, int ks) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, qd = lane & 3;
  struct Row {
    long long pix, off;  // pixel index (-1 past the image edge); element offset of (pixel, n0) in the [pixels, cout] outputs
    const __half *res, *res_lo;
    float r1x;
  };
  auto row_at = [&](const int i) {
    Row r;
    r.pix = row_pixel(p, b, y0, x0, tile_row(warp, lane, i));
    r.off = r.pix * p.cout + n0;
    r.res = p.res ? p.res + (p.res_batch_stride ? r.off : r.off - (long long)b * p.ho * p.wo * p.cout) : nullptr;
    r.res_lo = p.res_lo ? p.res_lo + (r.res - p.res) : nullptr;
    r.r1x = (p.rank1_x && r.pix >= 0) ? p.rank1_x[r.pix] : 0.f;
    return r;
  };
  // Column pair (8j + 2qd, +1) of row i; returns its ReLU'd value (the head's input).  `full`: the tile spans N existing channels of an even Cout,
  // so the per-column bounds check and the odd-Cout path drop out of the unrolled loop at compile time.
  auto pair = [&](auto full_t, const Row& r, const int i, const int j) {
    constexpr bool full = decltype(full_t)::value;
    const int col = 8 * j + 2 * qd;
    const int ch = n0 + col;
    if (!full && (col >= p.nt || ch >= p.cout)) return make_float2(0.f, 0.f);
    const float v0 = d[4 * j + 2 * i] * p.acc_scale, v1 = d[4 * j + 2 * i + 1] * p.acc_scale;
    // Unwanted addresses are formed from null bases, never used: `q ? q + e : nullptr` guards spill (N >= 128).
    const long long e = r.off + col;
    if (full || p.cout % 2 == 0) {  // both channels exist and the pair is 4-byte aligned in the fp16 outputs
      const float2 v = pair_value(p, v0, v1, ks == 0, s.bias + ch, s.r1w + ch, r.r1x, r.res + col, r.res_lo + col);
      const float2 a = relu2(v);
      pair_store(p, v, a, p.out_raw + e, p.out_raw_lo + e, p.out_relu + e, p.out_relu_lo + e, p.out_relu_lo8 + e);
      if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + ks * p.f32_split_stride + e) = v;
      return a;
    }
    // odd Cout (e.g. 1, 129): element by element
    return relu2(make_float2(finish_scalar(p, v0, ch, e, r.res, r.res_lo, col, r.r1x, ks),
                             ch + 1 < p.cout ? finish_scalar(p, v1, ch + 1, e + 1, r.res, r.res_lo, col + 1, r.r1x, ks) : v1));
  };
  if constexpr (HEAD) {
    // The host admits the head only when the tile is the whole Cout and exactly N wide, so every column pair takes the
    // full-width path.  Column pair outer, row inner: a pair's weights are loaded once for both rows.
    const Row rows[2] = {row_at(0), row_at(1)};
    float hacc[2][kMaxHead] = {};
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      float w[2 * kMaxHead];
      head_weights(s.head, j, qd, w);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (rows[i].pix < 0) continue;
        const float2 a = pair(std::true_type{}, rows[i], i, j);
        head_add(hacc[i], w, a.x, a.y);
      }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) head_store(p, hacc[i], rows[i].pix, qd);
  } else {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const Row r = row_at(i);
      if (r.pix >= 0) {
        if (p.cout % 2 == 0 && p.nt == N && n0 + N <= p.cout) {  // every tile of the wide layers
#pragma unroll
          for (int j = 0; j < N / 8; ++j) pair(std::true_type{}, r, i, j);
        } else {
#pragma unroll
          for (int j = 0; j < N / 8; ++j) pair(std::false_type{}, r, i, j);
        }
      }
    }
  }
}

// Gate form: the gated hidden-state update of the sensory updaters.  The channel tile is [forget | update | new] x 64
// for hidden channels hc0 .. hc0+63 (modules.py:145-149): the three gates of hidden channel c sit in columns c, 64 + c,
// 128 + c, i.e. in the same thread.
__device__ __forceinline__ void epilogue_gates(const Params& p, const Smem& s, const float (&d)[96], int b, int y0,
                                               int x0, int n0) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, qd = lane & 3;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const long long pix = row_pixel(p, b, y0, x0, tile_row(warp, lane, i));
    if (pix >= 0) {
      const int hc0 = (n0 / 192) * 64;
      const long long hoff = pix * p.gate_c + hc0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 8 * j + 2 * qd;
        const float2 hp = __half22float2(*reinterpret_cast<const __half2*>(p.gate_h + hoff + c));
        float o[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float f = sigmoid_fast(d[4 * j + 2 * i + e] + s.bias[n0 + c + e]);
          const float uu = sigmoid_fast(d[4 * (j + 8) + 2 * i + e] + s.bias[n0 + 64 + c + e]);
          const float n = tanh_fast(d[4 * (j + 16) + 2 * i + e] + s.bias[n0 + 128 + c + e]);
          o[e] = f * (e ? hp.y : hp.x) * (1.f - uu) + uu * n;
        }
        *reinterpret_cast<__half2*>(p.gate_out + hoff + c) = __floats2half2_rn(o[0], o[1]);
      }
    }
  }
}

// N: wgmma width (>= p.nt; columns past p.nt are never stored).
template <int N, int EPI>
__global__ void __launch_bounds__(THREADS, 1)
conv_kernel(const __grid_constant__ Maps maps, const __grid_constant__ Params p) {
  constexpr bool HEAD = EPI == EPI_HEAD;
  // 1024-byte alignment (128B swizzle atoms) comes from the declaration: deriving an aligned pointer through an
  // integer cast would make the compiler lose the shared address space (generic LD/ST instead of LDS/STS).
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + RING_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  float* s_head = reinterpret_cast<float*>(smem + RING_BYTES + 256);  // [128 pairs][kHeadPairStride] fused-head weights
  float* s_bias = s_head + HEAD_BYTES / 4;                            // [kMaxBias] bias of every output channel
  float* s_r1w = s_bias + kMaxBias;                                   // [kMaxRank1] rank-1 column

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int k8 = (p.taps - p.taps16) * p.cblocks8;  // fp8 correction k-iterations come first ...
  const int k_iters = k8 + p.taps16 * p.cblocks;     // ... then the fp16 ones
  const uint32_t stage_tx = A_BYTES + p.nt * BK * 2;

  if (warp == 8 && lane == 0) {
    for (int i = 0; i < 8; ++i) tma_prefetch_desc(&maps.act[i]);
    tma_prefetch_desc(&maps.wgt);
    tma_prefetch_desc(&maps.act8);
    tma_prefetch_desc(&maps.wgt8);
    // empty[]: every consumer thread arrives once the wgmma reading the stage have completed (a release by one thread
    // per warpgroup behind a branch puts the wgmma next to a divergent path, which makes ptxas serialize them)
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONSUMER_THREADS); }
    fence_barrier_init();
  }
  {  // bias (and the rank-1 column) of the whole layer: read once per CTA instead of once per tile from global memory
    const int cout_pad = p.n_tiles * p.nt;
    for (int i = threadIdx.x; i < cout_pad; i += THREADS) s_bias[i] = p.bias[i];
    if (p.rank1_w)
      for (int i = threadIdx.x; i < cout_pad; i += THREADS) s_r1w[i] = p.rank1_w[i];
  }
  __syncthreads();

  if (warp >= 8) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == CONSUMER_THREADS) {
      int stage = 0;
      uint32_t phase = 0;
      for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
        int b, y0, x0, n0, ks;
        tile_decode(u, p, b, y0, x0, n0, ks);
        const int k_lo = ks * p.k_per_split, k_hi = min(k_iters, k_lo + p.k_per_split);
        // flat tiles: the first pixel's filter-window origin
        const int fy = p.flat_wo ? x0 / p.flat_wo : 0, fx = x0 - fy * p.flat_wo - p.pad;
        // one k-iteration: activation box of tap t / channel block cb (+ the matching weight columns) into `stage`
        auto issue = [&](const int t, const int cb, const bool f8) {
          const int ch = f8 ? cb * 128 : cb * BK;
          const CUtensorMap* am = f8 ? &maps.act8 : &maps.act[p.tap_map[t]];
          const int wcol = f8 ? (p.tap_w[t] * p.cblocks8 + cb) * 128 : (p.tap_w[t] * p.cblocks + cb) * BK;
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], stage_tx);
          if (p.flat_wo) {
            const int c[4] = {ch, fx, fy - p.pad, b};  // (channel, x, y, image)
            tma_load_im2col_4d(sA + stage * A_BYTES, am, &full[stage], c, (uint16_t)(p.tap_dx[t] + p.pad),
                               (uint16_t)(p.tap_dy[t] + p.pad));
          } else {
            const int c[5] = {ch, x0 + p.tap_dx[t], y0 + p.tap_dy[t], b, 0};  // (channel, x, y, image, 1)
            tma_load_5d(sA + stage * A_BYTES, am, &full[stage], c);
          }
          tma_load_2d(sB + stage * B_BYTES_MAX, f8 ? &maps.wgt8 : &maps.wgt, &full[stage], wcol, n0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        };
        for (int t = p.taps16; t < p.taps; ++t)  // fp8 correction entries first (never combined with split-K)
          for (int cb = 0; cb < p.cblocks8; ++cb) issue(t, cb, true);
        for (int t = k_lo / p.cblocks; t < p.taps16 && t * p.cblocks < k_hi; ++t)
          for (int cb = max(0, k_lo - t * p.cblocks); cb < p.cblocks && t * p.cblocks + cb < k_hi; ++cb) issue(t, cb, false);
        if (p.staged) {  // one stage per 64-channel chunk: its residual box, or a reservation for the outputs
          const uint32_t res_tx = (p.res ? A_BYTES : 0) + (p.res_lo ? A_BYTES : 0);
          for (int n = 0; n < p.nt; n += 64) {
            mbar_wait(&empty[stage], phase ^ 1);
            if (res_tx) {
              const int c[5] = {n0 + n, x0, y0, p.res_batch_stride ? b : 0, 0};
              mbar_expect_tx(&full[stage], res_tx);
              if (p.res) tma_load_5d(sA + stage * A_BYTES, &maps.res, &full[stage], c);
              if (p.res_lo) tma_load_5d(sB + stage * B_BYTES_MAX, &maps.res_lo, &full[stage], c);
            } else {
              mbar_arrive(&full[stage]);
            }
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ---------------------------------------------------------------- consumers: warpgroup wg owns pixels wg*64 .. +63
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2;
  if constexpr (HEAD) {  // stage the head weights once per CTA, zero padded
    for (int i = threadIdx.x; i < HEAD_BYTES / 4; i += CONSUMER_THREADS) {
      const int pr = i / kHeadPairStride, k = i - pr * kHeadPairStride;
      const int t = k / 2, ch = 2 * pr + (k & 1);
      s_head[i] = (t < p.head_n && ch < p.cout) ? p.head_w[t * p.cout + ch] : 0.f;
    }
    named_bar_sync(1, CONSUMER_THREADS);
  }
  const uint32_t a_off = wg * 64 * 128;  // this warpgroup's 64 rows of the A tile (8 swizzle atoms)
  const Smem s = {sA, sB, full, empty, s_head, s_bias, s_r1w};
  float d[N / 2];
  int stage = 0;
  uint32_t phase = 0;
  for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
    int b, y0, x0, n0, ks;
    tile_decode(u, p, b, y0, x0, n0, ks);
    const int k_lo = ks * p.k_per_split;
    const int my_k = min(k_iters, k_lo + p.k_per_split) - k_lo;
    const int my_k8 = min(my_k, max(0, k8 - k_lo));  // the e4m3 k-iterations of this unit come first
    // k-iterations [ki0, ki1), all of one operand kind.  The kind is a template argument so that no wgmma sits in a
    // branch: ptxas then keeps one wgmma group in flight instead of draining each before the next.  A stage is
    // released once wgmma_wait<1> shows the group that read it has completed.
    auto k_loop = [&](auto f8, const int ki0, const int ki1) {
      for (int ki = ki0; ki < ki1; ++ki) {
        mbar_wait(&full[stage], phase);
        const uint32_t a_addr = smem_u32(sA + stage * A_BYTES) + a_off;
        const uint32_t b_addr = smem_u32(sB + stage * B_BYTES_MAX);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {  // 32 bytes of the 128-byte rows each: fp16 K = 16, e4m3 K = 32
          if constexpr (decltype(f8)::value)
            wgmma_e4m3<N>(d, wgmma_desc_sw128(a_addr + k * 32), wgmma_desc_sw128(b_addr + k * 32), (ki | k) != 0);
          else
            wgmma_f16<N>(d, wgmma_desc_sw128(a_addr + k * 32), wgmma_desc_sw128(b_addr + k * 32), (ki | k) != 0);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (ki > 0) mbar_arrive(&empty[stage == 0 ? STAGES - 1 : stage - 1]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    };
    k_loop(std::true_type{}, 0, my_k8);
    k_loop(std::false_type{}, my_k8, my_k);
    wgmma_wait<0>();
    wgmma_fence_regs(d);
    mbar_arrive(&empty[stage == 0 ? STAGES - 1 : stage - 1]);  // the stage of the last k-iteration (my_k >= 1)

    if constexpr (EPI == EPI_GATES)
      epilogue_gates(p, s, d, b, y0, x0, n0);
    else if (p.staged)
      epilogue_staged<N, HEAD>(maps, p, s, d, stage, phase, b, y0, x0, n0);
    else
      epilogue_regs<N, HEAD>(p, s, d, b, y0, x0, n0, ks);
  }
}

}  // namespace conv
}  // namespace b200

using namespace b200;

// Staged epilogue plan (p.staged, output regions, tensor maps; ho, wo, p.th, p.tw as the kernel sees them, i.e. 1, Ho * Wo,
// 1, 128 for flat tiles): every tile spans exactly N existing channels, fp16 / e4m3
// outputs that fit the three regions of a stage, 16-byte aligned operands (TMA).  DEVA_B200_CONV_EPI=regs keeps the
// per-thread epilogue (A/B comparisons); DEVA_B200_CONV_EPI=staged refuses a launch that cannot take the staged one.
static int plan_staged(const deva_b200_conv_desc& d, int ho, int wo, int n_mma, conv::Params& p, conv::Maps& maps) {
  using namespace conv;
  const char* err = nullptr;
  const char* env = getenv("DEVA_B200_CONV_EPI");
  const bool regs = env && strcmp(env, "regs") == 0, must = env && strcmp(env, "staged") == 0;
  auto aligned = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  const bool pool = d.out_pool4 != nullptr;
  // fp16 regions in order: raw (also staged, unstored, when only its pool is wanted), raw_lo, relu, relu_lo
  const void* outs[4] = {d.out_raw, d.out_raw_lo, d.out_relu, d.out_relu_lo};
  const bool used[4] = {d.out_raw || pool, d.out_raw_lo != nullptr, d.out_relu != nullptr, d.out_relu_lo != nullptr};
  int n16 = 0;
  for (int k = 0; k < 4; ++k) n16 += used[k] ? 1 : 0;
  // the e4m3 region (64-byte rows) must not overlay a residual half that other threads have yet to read
  const int r_lo8 = std::max({n16, d.res ? 1 : 0, d.res_lo ? 2 : 0});
  // a low-order part without its fp16 output is written by neither epilogue form, so the staged one must not store it
  const bool ok = !regs && !p.gate_out && p.ksplit == 1 && !d.out_f32 && d.nt == n_mma && d.cout == d.cout_pad &&
                  (!d.res_lo || d.res) && !(d.out_raw_lo && !d.out_raw) && !(d.out_relu_lo && !d.out_relu) &&
                  aligned(d.res) && aligned(d.res_lo) && aligned(d.out_raw) && aligned(d.out_raw_lo) &&
                  aligned(d.out_relu) && aligned(d.out_relu_lo) && aligned(d.out_relu_lo8) && aligned(d.out_pool4) &&
                  (d.out_relu_lo8 ? r_lo8 <= 2 : n16 <= 3);
  B200_REQUIRE(ok || !(must || pool), "conv: %s needs the staged epilogue (full-width channel tiles, cout == cout_pad, "
               "no fp32 / split-K / gate outputs, outputs that fit a ring stage)%s", pool ? "out_pool4" : "DEVA_B200_CONV_EPI=staged",
               regs ? ", which DEVA_B200_CONV_EPI=regs turns off" : "");
  B200_REQUIRE(!pool || (d.th % 4 == 0 && d.tw % 4 == 0 && ho % 4 == 0 && wo % 4 == 0),
               "conv: out_pool4 needs th, tw (%d, %d) and ho, wo (%d, %d) multiples of 4", d.th, d.tw, ho, wo);
  if (ok) {
    const long long cstr = d.cout, wstr = (long long)wo * d.cout, bstr = (long long)ho * wo * d.cout;
    signed char* regs_of[4] = {&p.reg_raw, &p.reg_raw_lo, &p.reg_relu, &p.reg_relu_lo};
    int rc = 0, k16 = 0;
    for (int k = 0; k < 4; ++k) {
      if (!used[k]) continue;
      *regs_of[k] = (signed char)k16;
      if (outs[k]) {
        rc |= make_tmap_act5(&maps.out[k16], outs[k], d.cout, wo, ho, d.batch, cstr, wstr, bstr, p.tw, p.th, &err);
        p.store_mask |= 1 << k16;
      }
      ++k16;
    }
    if (d.out_relu_lo8) {
      p.reg_lo8 = (signed char)r_lo8;
      rc |= make_tmap_act5_u8(&maps.out[r_lo8], d.out_relu_lo8, d.cout, wo, ho, d.batch, cstr, wstr, bstr, 64, p.tw, p.th,
                              &err);
      p.store_mask |= 1 << r_lo8;
    }
    const int rb = d.res_broadcast ? 1 : d.batch;
    if (d.res) rc |= make_tmap_act5(&maps.res, d.res, d.cout, wo, ho, rb, cstr, wstr, bstr, p.tw, p.th, &err);
    if (d.res_lo) rc |= make_tmap_act5(&maps.res_lo, d.res_lo, d.cout, wo, ho, rb, cstr, wstr, bstr, p.tw, p.th, &err);
    if (rc) {
      set_error("conv: %s", err ? err : "epilogue tensor maps");
      return 3;
    }
    p.staged = 1;
    p.out_pool4 = reinterpret_cast<__half*>(d.out_pool4);
  }
  return 0;
}

extern "C" {

// The descriptor is read on the host only: the kernel receives the Params built from it.
DEVA_B200_API int deva_b200_conv2d(const deva_b200_conv_desc* desc, deva_stream_t stream) {
  using namespace conv;
  const deva_b200_conv_desc& d = *desc;
  B200_REQUIRE(d.cin_pad % 64 == 0 && d.cin_pad >= 64, "conv: cin_pad %d must be a multiple of 64", d.cin_pad);
  B200_REQUIRE(d.stride == 1 || d.stride == 2, "conv: stride %d unsupported", d.stride);
  B200_REQUIRE(d.kh == d.kw && (d.kh == 1 || d.kh == 3), "conv: %dx%d filter unsupported here", d.kh, d.kw);
  B200_REQUIRE(d.nt % 32 == 0 && d.nt >= 32 && d.nt <= 256 && d.cout_pad % d.nt == 0, "conv: bad channel tile %d", d.nt);
  const bool flat = d.th == 0;  // flat tiles: 128 consecutive pixels of one image (th = 0, tw = 128)
  B200_REQUIRE(flat ? d.tw == 128 : (d.th > 0 && d.tw * d.th == 128 && d.tw <= 256 && d.th <= 256),
               "conv: spatial tile %dx%d must cover 128 pixels (or be 0 x 128: flat tiles)", d.th, d.tw);
  B200_REQUIRE(!flat || (d.stride == 1 && !d.out_pool4),
               "conv: flat tiles need stride 1 (got %d) and no out_pool4 (its windows need rectangular tiles)", d.stride);
  B200_REQUIRE(d.cout_pad <= conv::kMaxBias && (!d.rank1_w || d.cout_pad <= conv::kMaxRank1),
               "conv: Cout_pad %d exceeds the shared-memory bias table (%d; %d with a rank-1 input)", d.cout_pad, conv::kMaxBias,
               conv::kMaxRank1);
  const int pad = d.kh / 2;
  const int ho = (d.h + 2 * pad - d.kh) / d.stride + 1;
  const int wo = (d.w + 2 * pad - d.kw) / d.stride + 1;
  Maps maps;
  Params p{};
  const char* err = nullptr;
  const int ktaps = d.kh * d.kw;
  B200_REQUIRE(!(d.x2 && d.x_lo), "conv: x2 (concat) and x_lo (split precision) are exclusive");
  // activation sources and the (source, weight group) passes of the K loop
  const void* srcs[2] = {d.x, d.x2 ? d.x2 : d.x_lo};
  const int n_src = (d.x2 || d.x_lo) ? 2 : 1;
  int pass_src[3] = {0, 0, 0}, pass_w[3] = {0, 0, 0}, n_pass = 1, w_groups = 1;
  if (d.x2) { n_pass = 2; pass_src[1] = 1; pass_w[1] = 1; w_groups = 2; }          // cat[x, x2] . [W0 | W1]
  B200_REQUIRE(d.split_mode == 0 || d.split_mode == 2 || d.split_mode == 3, "conv: split_mode %d unknown", d.split_mode);
  B200_REQUIRE(d.split_mode != 2 || (!d.x_lo && !d.x2), "conv: split_mode 2 (weight hi/lo) takes a single input");
  B200_REQUIRE(d.split_mode != 3 || (d.x_lo8 && d.w8_packed && !d.x_lo && !d.x2 && d.stride == 1 && d.cin_pad % 128 == 0 &&
                                     d.ksplit <= 1),
               "conv: split_mode 3 (fp8 correction pass) needs x_lo8 + w8_packed, stride 1, cin_pad %% 128 == 0, no x_lo / x2 / ksplit");
  if (d.split_mode == 2) { n_pass = 2; pass_src[1] = 0; pass_w[1] = 1; w_groups = 2; }  // X.Wh + X.Wl
  else if (d.x_lo) { n_pass = 3; pass_src[1] = 1; pass_w[1] = 0; pass_src[2] = 0; pass_w[2] = 1; w_groups = 2; }  // Xh.Wh + Xl.Wh + Xh.Wl
  p.taps16 = ktaps * n_pass;
  p.taps = p.taps16 + (d.split_mode == 3 ? ktaps : 0);  // fp8 correction: one more pass, 128 channels per k-iteration
  p.cblocks8 = d.split_mode == 3 ? d.cin_pad / 128 : 0;
  p.acc_scale = d.acc_scale != 0.f ? d.acc_scale : 1.f;
  p.out_relu_lo8 = reinterpret_cast<uint8_t*>(d.out_relu_lo8);
  B200_REQUIRE(p.taps <= kMaxTaps, "conv: too many k-entries (%d)", p.taps);
  const int phases = d.stride == 1 ? 1 : 4;
  bool built[8] = {false, false, false, false, false, false, false, false};
  for (int sidx = 0; sidx < n_src; ++sidx) {
    const __half* xs = reinterpret_cast<const __half*>(srcs[sidx]);
    for (int ph = 0; ph < phases; ++ph) {
      const int py = ph / 2, px = ph % 2;
      int rc;
      if (flat) {
        rc = make_tmap_im2col4(&maps.act[sidx * 4], TmapType::F16, xs, d.cin_pad, d.w, d.h, d.batch, 64, pad, &err);
        built[sidx * 4] = true;
      } else if (d.stride == 1) {
        rc = make_tmap_act5(&maps.act[sidx * 4], xs, d.cin_pad, d.w, d.h, d.batch, (long long)d.cin_pad,
                            (long long)d.w * d.cin_pad, (long long)d.h * d.w * d.cin_pad, d.tw, d.th, &err);
        built[sidx * 4] = true;
      } else {
        // phase (py, px): rows y = 2*i + py, cols x = 2*j + px of the same NHWC buffer
        const int hp = (d.h - py + 1) / 2, wp = (d.w - px + 1) / 2;
        if (hp <= 0 || wp <= 0) continue;
        rc = make_tmap_act5(&maps.act[sidx * 4 + ph], xs + ((long long)py * d.w + px) * d.cin_pad, d.cin_pad, wp, hp,
                            d.batch, 2ll * d.cin_pad, 2ll * d.w * d.cin_pad, (long long)d.h * d.w * d.cin_pad, d.tw,
                            d.th, &err);
        built[sidx * 4 + ph] = true;
      }
      if (rc) {
        set_error("conv: %s", err ? err : "tensor map");
        return 3;
      }
    }
  }
  for (int i = 1; i < 8; ++i)  // unused slots still get prefetched: point them at a valid descriptor
    if (!built[i]) maps.act[i] = maps.act[0];
  for (int t = 0; t < p.taps; ++t) {
    const int pass = t < p.taps16 ? t / ktaps : 0, kt = t % ktaps;
    const int oy = kt / d.kw - pad, ox = kt % d.kw - pad;  // input offset relative to stride*yo, stride*xo
    int ph = 0, dy = oy, dx = ox;
    if (d.stride == 2) {
      const int py = ((oy % 2) + 2) % 2, px = ((ox % 2) + 2) % 2;
      ph = py * 2 + px;
      dy = (oy - py) / 2;
      dx = (ox - px) / 2;
      // An input one row (column) high (wide) has no odd-row (odd-column) phase: every tap of that phase reads
      // padding, but its map slot holds phase 0's map.  Its box is moved wholly above (left of) the image instead, so
      // that TMA fills it with zeros: the output is then one row (column) high, y0 = 0 (x0 = 0).
      if (py >= d.h) dy = -d.th;
      if (px >= d.w) dx = -d.tw;
    }
    p.tap_map[t] = (signed char)(pass_src[pass] * 4 + ph);
    p.tap_w[t] = (signed char)(t < p.taps16 ? pass_w[pass] * ktaps + kt : kt);
    p.tap_dy[t] = (signed char)dy;
    p.tap_dx[t] = (signed char)dx;
  }
  if (make_tmap_2d(&maps.wgt, TmapType::F16, d.w_packed, (uint64_t)w_groups * ktaps * d.cin_pad, d.cout_pad,
                   (uint64_t)w_groups * ktaps * d.cin_pad * 2, 64, d.nt, &err)) {
    set_error("conv: %s", err ? err : "weight tensor map");
    return 3;
  }
  p.batch = d.batch; p.ho = ho; p.wo = wo; p.cout = d.cout;
  if (flat) {  // see Params::flat_wo
    p.ho = 1; p.wo = ho * wo; p.th = 1; p.tw = 128;
    p.flat_wo = wo; p.pad = pad;
  } else {
    p.tw = d.tw; p.th = d.th;
  }
  p.tiles_x = ceil_div(p.wo, p.tw); p.tiles_y = ceil_div(p.ho, p.th);
  p.nt = d.nt; p.n_tiles = d.cout_pad / d.nt;
  p.cblocks = d.cin_pad / 64;
  p.m_tiles = p.batch * p.tiles_y * p.tiles_x;
  p.bias = d.bias;
  p.res = reinterpret_cast<const __half*>(d.res);
  p.res_lo = reinterpret_cast<const __half*>(d.res_lo);
  p.res_batch_stride = d.res_broadcast ? 0 : (long long)ho * wo * d.cout;
  p.rank1_w = d.rank1_w; p.rank1_x = d.rank1_x;
  p.out_raw = reinterpret_cast<__half*>(d.out_raw);
  p.out_relu = reinterpret_cast<__half*>(d.out_relu);
  p.out_f32 = d.out_f32;
  p.out_raw_lo = reinterpret_cast<__half*>(d.out_raw_lo);
  p.out_relu_lo = reinterpret_cast<__half*>(d.out_relu_lo);
  if (d.gate_out) {
    // the gates are evaluated on the unscaled accumulator (epilogue_gates)
    B200_REQUIRE(d.gate_h && d.nt == 192 && d.cout == d.cout_pad && d.cout % 192 == 0 && !d.head_w && !d.res && !d.rank1_w &&
                     !d.out_raw && !d.out_relu && !d.out_f32 && p.acc_scale == 1.f,
                 "conv: the gate epilogue needs nt == 192, cout = 3 * C with C %% 64 == 0 (got %d), acc_scale 1 and no other "
                 "outputs", d.cout);
    p.gate_h = reinterpret_cast<const __half*>(d.gate_h);
    p.gate_out = reinterpret_cast<__half*>(d.gate_out);
    p.gate_c = d.cout / 3;
  }
  if (d.head_w) {
    // the head epilogue has only the full-width column loop: one tile of exactly N = 64 / 128 / 192 / 256 channels
    B200_REQUIRE(d.cout == d.nt && d.cout_pad == d.nt && d.cout % 64 == 0 && d.cout <= 256 && d.head_n >= 1 &&
                     d.head_n <= kMaxHead && d.head_out,
                 "conv: fused head needs Cout (%d) = channel tile (%d) in {64, 128, 192, 256} and 1 <= head_n (%d) <= %d",
                 d.cout, d.nt, d.head_n, kMaxHead);
    p.head_w = d.head_w; p.head_out = d.head_out; p.head_n = d.head_n;
  }
  // wgmma width: the channel tile rounded up to one of four instantiations.  TMA fills only nt weight rows of a stage;
  // rows nt .. N-1 hold whatever an earlier stage left there, so columns nt .. N-1 of the accumulator are garbage and the
  // epilogue never stores them (col < p.nt).  The cost is up to half the MMA work of layers with a ragged tile
  // (Cout 1 -> N 64, Cout 129 -> nt 160 -> N 192); those layers are small.
  const int n_mma = d.nt <= 64 ? 64 : (d.nt <= 128 ? 128 : (d.nt <= 192 ? 192 : 256));
  const int epi = p.gate_out ? EPI_GATES : (p.head_w ? EPI_HEAD : EPI_PLAIN);
  void (*kern)(const Maps, const Params) = nullptr;
  if (epi == EPI_GATES) kern = conv_kernel<192, EPI_GATES>;
  else if (epi == EPI_HEAD)
    kern = n_mma == 64 ? conv_kernel<64, EPI_HEAD> : n_mma == 128 ? conv_kernel<128, EPI_HEAD>
         : n_mma == 192 ? conv_kernel<192, EPI_HEAD> : conv_kernel<256, EPI_HEAD>;
  else
    kern = n_mma == 64 ? conv_kernel<64, EPI_PLAIN> : n_mma == 128 ? conv_kernel<128, EPI_PLAIN>
         : n_mma == 192 ? conv_kernel<192, EPI_PLAIN> : conv_kernel<256, EPI_PLAIN>;
  static bool configured_dev[kMaxDevices] = {false};  // function attributes are per device
  bool& configured = configured_dev[device_slot()];
  if (!configured) {
    for (auto k : {conv_kernel<64, EPI_PLAIN>, conv_kernel<128, EPI_PLAIN>, conv_kernel<192, EPI_PLAIN>, conv_kernel<256, EPI_PLAIN>,
                   conv_kernel<64, EPI_HEAD>, conv_kernel<128, EPI_HEAD>, conv_kernel<192, EPI_HEAD>, conv_kernel<256, EPI_HEAD>,
                   conv_kernel<192, EPI_GATES>})
      B200_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    configured = true;
  }
  maps.act8 = maps.act[0];
  maps.wgt8 = maps.wgt;
  if (d.split_mode == 3) {
    const uint64_t k8 = (uint64_t)ktaps * d.cin_pad;  // bytes per weight row (cin_pad is a multiple of 128)
    if ((flat ? make_tmap_im2col4(&maps.act8, TmapType::U8, d.x_lo8, d.cin_pad, d.w, d.h, d.batch, 128, pad, &err)
              : make_tmap_act5_u8(&maps.act8, d.x_lo8, d.cin_pad, d.w, d.h, d.batch, (long long)d.cin_pad,
                                  (long long)d.w * d.cin_pad, (long long)d.h * d.w * d.cin_pad, 128, d.tw, d.th, &err)) ||
        make_tmap_2d(&maps.wgt8, TmapType::U8, d.w8_packed, k8, d.cout_pad, k8, 128, d.nt, &err)) {
      set_error("conv: %s", err ? err : "fp8 tensor maps");
      return 3;
    }
  }
  // split-K: fp32 output only
  p.ksplit = d.ksplit > 1 ? d.ksplit : 1;
  const int k_iters_total = p.taps16 * p.cblocks + (p.taps - p.taps16) * p.cblocks8;
  if (p.ksplit > 1) {
    B200_REQUIRE(d.out_f32 && !d.out_raw && !d.out_relu && !d.res && !d.rank1_w && !d.head_w && !d.gate_out,
                 "conv: split-K writes fp32 partial sums only (no residual / rank-1 / head / gates / fp16 outputs)");
    B200_REQUIRE(p.ksplit <= k_iters_total, "conv: ksplit %d exceeds the %d k-iterations", p.ksplit, k_iters_total);
  }
  p.k_per_split = (k_iters_total + p.ksplit - 1) / p.ksplit;
  p.ksplit = (k_iters_total + p.k_per_split - 1) / p.k_per_split;  // no empty trailing split
  p.f32_split_stride = (long long)d.batch * ho * wo * d.cout;
  if (const int rc = plan_staged(d, p.ho, p.wo, n_mma, p, maps)) return rc;
  const long long units = (long long)p.m_tiles * p.n_tiles * p.ksplit;
  B200_REQUIRE(units <= INT32_MAX, "conv: %lld work units", units);
  p.units = (int)units;
  const int grid = (int)(units < sm_count() ? units : sm_count());
  kern<<<grid, THREADS, SMEM_BYTES, S(stream)>>>(maps, p);
  B200_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
