// Segment Anything's automatic masks from the mask decoder's low-resolution logits (deva/ext/sam_masks.py, DESIGN §7).
// Sam.postprocess_masks upsamples each [lh, lw] logit map bilinearly to the [grid, grid] input grid, crops it to the
// input size [in_h, in_w] and upsamples that to the frame [out_h, out_w].  Everything the automatic generator keeps of
// those full-resolution maps is a handful of integers per mask, so the value of every frame pixel is evaluated here,
// in registers and shared memory, and never stored:
//   1. stats_kernel<false>: one CTA per (mask, band of frame rows).  The stage-1 rows the band reads are produced as
//      float32 into shared memory, then every frame pixel of the band is interpolated from them and compared with the
//      three cutoffs of calculate_stability_score and the mask threshold; counts and the box are reduced in the CTA
//      and added to the mask's seven int32 counters with one atomic each;
//   2. compact_kernel: stability = intersections / unions in float32, the predicted-IoU and stability filters, and
//      the kept masks' indices in ascending order;
//   3. rank_kernel, iou_mask_kernel, greedy_kernel: torchvision's CUDA nms, scores in a stable descending order;
//   4. stats_kernel<true>: the same two-stage values of the kept masks, thresholded and written as bool.
// Both interpolation stages use the arithmetic of ATen's CUDA upsample_bilinear2d (align_corners=False, an output size
// and no scale factor): scale = float(in) / out, source index scale * (dst + 0.5) - 0.5 clamped at 0, lambdas and the
// two-level weighted sum in the same order, so the values are torch's float32 values.
#include <stdint.h>

#include "common.h"
#include "scan.cuh"

namespace b200 {
namespace sam {

constexpr int kThreads = 256;
constexpr int kStageRows = 8;     // stage-1 rows held in shared memory at once
constexpr int kMaxGrid = 1024;    // longest stage-1 row
constexpr int kBandRows = 32;     // frame rows per CTA
constexpr int kStats = 7;         // per mask: > thr + offset, > thr - offset, > thr, x0, y0, x1, y1
constexpr int kNmsWord = 64;

struct Axis {
  int i0, i1;  // the two source indices
  float l0, l1;  // their weights
};

// ATen's area_pixel_compute_source_index (align_corners=False, not cubic) and the neighbours and lambdas of
// upsample_bilinear2d_out_frame.
__device__ __forceinline__ Axis axis(float scale, int dst, int in) {
  float r = scale * (dst + 0.5f) - 0.5f;
  r = r < 0 ? 0.f : r;
  Axis a;
  a.i0 = (int)r;
  a.i1 = a.i0 + ((a.i0 < in - 1) ? 1 : 0);
  a.l1 = r - a.i0;
  a.l0 = 1.f - a.l1;
  return a;
}

__device__ __forceinline__ float lerp2(const Axis& h, const Axis& w, float v00, float v01, float v10, float v11) {
  return h.l0 * (w.l0 * v00 + w.l1 * v01) + h.l1 * (w.l0 * v10 + w.l1 * v11);
}

struct Shape {
  int lh, lw, grid, in_h, in_w, out_h, out_w;
  float s1h, s1w, s2h, s2w;  // float(in) / out of each stage
};

// The CTA's counts and box -> the mask's counters: warp shuffles, one shared atomic per warp, one global atomic per field.
__device__ __forceinline__ void reduce_into(int32_t* st, int* red, int hi, int lo, int mid, int x0, int y0, int x1,
                                            int y1) {
  for (int o = 16; o; o >>= 1) {
    hi += __shfl_xor_sync(0xffffffffu, hi, o);
    lo += __shfl_xor_sync(0xffffffffu, lo, o);
    mid += __shfl_xor_sync(0xffffffffu, mid, o);
    x0 = min(x0, __shfl_xor_sync(0xffffffffu, x0, o));
    y0 = min(y0, __shfl_xor_sync(0xffffffffu, y0, o));
    x1 = max(x1, __shfl_xor_sync(0xffffffffu, x1, o));
    y1 = max(y1, __shfl_xor_sync(0xffffffffu, y1, o));
  }
  if (threadIdx.x < kStats) red[threadIdx.x] = threadIdx.x < 3 ? 0 : (threadIdx.x < 5 ? INT32_MAX : -1);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&red[0], hi), atomicAdd(&red[1], lo), atomicAdd(&red[2], mid);
    atomicMin(&red[3], x0), atomicMin(&red[4], y0), atomicMax(&red[5], x1), atomicMax(&red[6], y1);
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    if (red[threadIdx.x]) atomicAdd(&st[threadIdx.x], red[threadIdx.x]);
  } else if (threadIdx.x < 5) {
    atomicMin(&st[threadIdx.x], red[threadIdx.x]);
  } else if (threadIdx.x < kStats) {
    atomicMax(&st[threadIdx.x], red[threadIdx.x]);
  }
}

template <bool kWrite>
__global__ void __launch_bounds__(kThreads) stats_kernel(const float* __restrict__ logits, const int64_t* __restrict__ sel,
                                                         Shape p, const float* __restrict__ iou, float iou_thresh,
                                                         float thr_hi, float thr_lo, float thr, int32_t* __restrict__ stats,
                                                         uint8_t* __restrict__ out) {
  __shared__ float s1[kStageRows][kMaxGrid];
  __shared__ int red[kStats];
  const int m = blockIdx.y;
  if (!kWrite && iou && !(iou[m] > iou_thresh)) return;  // filtered by predicted IoU: counters stay at their init
  const float* src = logits + (size_t)(kWrite ? sel[m] : m) * p.lh * p.lw;
  const int y_begin = blockIdx.x * kBandRows, y_end = min(p.out_h, y_begin + kBandRows);
  int hi = 0, lo = 0, mid = 0, x0 = INT32_MAX, y0 = INT32_MAX, x1 = -1, y1 = -1;
  for (int y = y_begin; y < y_end;) {
    // stage-1 rows [r_lo, r_hi] feed frame rows [y, y_last]
    const int r_lo = axis(p.s2h, y, p.in_h).i0;
    int y_last = y;
    while (y_last + 1 < y_end && axis(p.s2h, y_last + 1, p.in_h).i1 - r_lo < kStageRows) ++y_last;
    const int r_hi = axis(p.s2h, y_last, p.in_h).i1;
    for (int k = threadIdx.x; k < (r_hi - r_lo + 1) * p.in_w; k += kThreads) {
      const int r = r_lo + k / p.in_w, c = k % p.in_w;
      const Axis h = axis(p.s1h, r, p.lh), w = axis(p.s1w, c, p.lw);
      const float* a = src + (size_t)h.i0 * p.lw;
      const float* b = src + (size_t)h.i1 * p.lw;
      s1[r - r_lo][c] = lerp2(h, w, __ldg(a + w.i0), __ldg(a + w.i1), __ldg(b + w.i0), __ldg(b + w.i1));
    }
    __syncthreads();
    for (int yy = y; yy <= y_last; ++yy) {
      const Axis h = axis(p.s2h, yy, p.in_h);
      const float* a = s1[h.i0 - r_lo];
      const float* b = s1[h.i1 - r_lo];
      uint8_t* row = kWrite ? out + ((size_t)m * p.out_h + yy) * p.out_w : nullptr;
      for (int x = threadIdx.x; x < p.out_w; x += kThreads) {
        const Axis w = axis(p.s2w, x, p.in_w);
        const float v = lerp2(h, w, a[w.i0], a[w.i1], b[w.i0], b[w.i1]);
        if (kWrite) {
          row[x] = v > thr;
        } else {
          hi += v > thr_hi;
          lo += v > thr_lo;
          if (v > thr) {
            ++mid;
            x0 = min(x0, x), x1 = max(x1, x), y0 = min(y0, yy), y1 = max(y1, yy);
          }
        }
      }
    }
    __syncthreads();
    y = y_last + 1;
  }
  if constexpr (!kWrite) reduce_into(stats + (size_t)m * kStats, red, hi, lo, mid, x0, y0, x1, y1);
}

__global__ void init_kernel(int n, int32_t* __restrict__ stats) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * kStats) return;
  const int f = (int)(i % kStats);
  stats[i] = f < 3 ? 0 : (f < 5 ? INT32_MAX : -1);
}

// One CTA: stability, the two filters, the box of every mask (batched_mask_to_box: [0, 0, 0, 0] when empty) and the
// ascending list of kept masks, kept[0] = their number.
__global__ void __launch_bounds__(1024) compact_kernel(const int32_t* __restrict__ stats, const float* __restrict__ iou,
                                                       int n, float iou_thresh, float stability_thresh,
                                                       float* __restrict__ stability, int64_t* __restrict__ boxes,
                                                       int32_t* __restrict__ kept) {
  __shared__ int warp_sums[32];
  int carry = 0;
  for (int base = 0; base < n; base += blockDim.x) {
    const int i = base + threadIdx.x;
    int keep = 0;
    if (i < n) {
      const int32_t* st = stats + (size_t)i * kStats;
      const float s = (float)st[0] / (float)st[1];
      stability[i] = s;
      keep = (!iou || iou[i] > iou_thresh) && (!(stability_thresh > 0.f) || s >= stability_thresh);
      const bool any = st[2] > 0;
      boxes[4 * i + 0] = any ? st[3] : 0;
      boxes[4 * i + 1] = any ? st[4] : 0;
      boxes[4 * i + 2] = any ? st[5] : 0;
      boxes[4 * i + 3] = any ? st[6] : 0;
    }
    int total;
    const int at = block_exclusive_scan(keep, warp_sums, total);
    if (keep) kept[1 + carry + at] = i;
    carry += total;
  }
  if (threadIdx.x == 0) kept[0] = carry;
}

// order[rank] = i, rank = the number of scores before i in a stable descending sort.
__global__ void rank_kernel(const float* __restrict__ scores, int n, int32_t* __restrict__ order) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float s = scores[i];
  int rank = 0;
  for (int j = 0; j < n; ++j) {
    const float t = scores[j];
    rank += (t > s) || (t == s && j < i);
  }
  order[rank] = i;
}

// torchvision's devIoU on the sorted boxes: bit j of row i's word (j / 64) is set when j > i overlaps i above thresh.
__global__ void iou_mask_kernel(const float* __restrict__ boxes, const int32_t* __restrict__ order, int n, float thresh,
                                unsigned long long* __restrict__ mask) {
  const int words = (n + kNmsWord - 1) / kNmsWord;
  const int i = blockIdx.x * blockDim.x + threadIdx.x, word = blockIdx.y;
  if (i >= n) return;
  const float* a = boxes + 4 * (size_t)order[i];
  unsigned long long bits = 0;
  for (int k = 0; k < kNmsWord; ++k) {
    const int j = word * kNmsWord + k;
    if (j <= i || j >= n) continue;
    const float* b = boxes + 4 * (size_t)order[j];
    const float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
    const float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
    const float width = fmaxf(right - left, 0.f), height = fmaxf(bottom - top, 0.f);
    const float inter = __fmul_rn(width, height);
    const float sa = __fmul_rn(a[2] - a[0], a[3] - a[1]);
    const float sb = __fmul_rn(b[2] - b[0], b[3] - b[1]);
    if (__fdiv_rn(inter, sa + sb - inter) > thresh) bits |= 1ull << k;
  }
  mask[(size_t)i * words + word] = bits;
}

// One CTA walks the sorted boxes: a box not yet suppressed is kept and suppresses its row of the mask.
__global__ void __launch_bounds__(1024) greedy_kernel(const unsigned long long* __restrict__ mask,
                                                      const int32_t* __restrict__ order, int n,
                                                      int64_t* __restrict__ keep, int32_t* __restrict__ n_keep) {
  extern __shared__ unsigned long long removed[];
  const int words = (n + kNmsWord - 1) / kNmsWord;
  for (int w = threadIdx.x; w < words; w += blockDim.x) removed[w] = 0;
  __syncthreads();
  int kept = 0;
  for (int i = 0; i < n; ++i) {
    const bool live = !((removed[i / kNmsWord] >> (i % kNmsWord)) & 1);
    __syncthreads();
    if (!live) continue;
    if (threadIdx.x == 0) keep[kept] = order[i];
    ++kept;
    for (int w = i / kNmsWord + threadIdx.x; w < words; w += blockDim.x) removed[w] |= mask[(size_t)i * words + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *n_keep = kept;
}

inline bool shape(int lh, int lw, int grid, int in_h, int in_w, int out_h, int out_w, Shape* p) {
  if (lh < 1 || lw < 1 || grid < 1 || grid > kMaxGrid || in_h < 1 || in_w < 1 || in_h > grid || in_w > grid ||
      out_h < 1 || out_w < 1 || (long long)out_h * out_w >= (1ll << 31) || out_h > 65535 * kBandRows)
    return false;
  *p = Shape{lh, lw, grid, in_h, in_w, out_h, out_w, (float)lh / grid, (float)lw / grid, (float)in_h / out_h,
             (float)in_w / out_w};
  return true;
}

}  // namespace sam
}  // namespace b200

using namespace b200;

DEVA_B200_API int deva_b200_sam_mask_stats(const float* logits, int n, int lh, int lw, int grid, int in_h, int in_w,
                                           int out_h, int out_w, const float* iou, float iou_thresh, float thr_hi,
                                           float thr_lo, float thr, int32_t* stats, deva_stream_t stream) {
  sam::Shape p;
  B200_REQUIRE(sam::shape(lh, lw, grid, in_h, in_w, out_h, out_w, &p),
               "sam_mask_stats: logits %d x %d, grid %d, input %d x %d, frame %d x %d out of range", lh, lw, grid, in_h,
               in_w, out_h, out_w);
  B200_REQUIRE(n >= 0 && n <= 65535, "sam_mask_stats: %d masks, expected 0 to 65535", n);
  if (n == 0) return 0;
  B200_REQUIRE(logits && stats, "sam_mask_stats: null pointer");
  cudaStream_t s = S(stream);
  sam::init_kernel<<<ceil_div((long long)n * sam::kStats, 256), 256, 0, s>>>(n, stats);
  B200_LAUNCH_CHECK();
  const dim3 blocks((unsigned)ceil_div(out_h, sam::kBandRows), (unsigned)n);
  sam::stats_kernel<false><<<blocks, sam::kThreads, 0, s>>>(logits, nullptr, p, iou, iou_thresh, thr_hi, thr_lo, thr,
                                                            stats, nullptr);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_sam_mask_compact(const int32_t* stats, const float* iou, int n, float iou_thresh,
                                             float stability_thresh, float* stability, int64_t* boxes, int32_t* kept,
                                             deva_stream_t stream) {
  B200_REQUIRE(n >= 0 && stats && stability && boxes && kept, "sam_mask_compact: bad arguments (n = %d)", n);
  sam::compact_kernel<<<1, 1024, 0, S(stream)>>>(stats, iou, n, iou_thresh, stability_thresh, stability, boxes, kept);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API size_t deva_b200_sam_nms_workspace_bytes(int n) {
  if (n < 0) return 0;
  Carver<16> c{nullptr};
  c.take<int32_t>(n);
  c.take<unsigned long long>((long long)n * ceil_div(n, sam::kNmsWord));
  return c.bytes;
}

DEVA_B200_API int deva_b200_sam_nms(const float* boxes, const float* scores, int n, float iou_thresh, void* workspace,
                                    int64_t* keep, int32_t* n_keep, deva_stream_t stream) {
  const int words = ceil_div(n, sam::kNmsWord);
  B200_REQUIRE(n >= 0 && (size_t)words * 8 <= 200 * 1024, "sam_nms: %d boxes, expected at most %d", n,
               200 * 1024 / 8 * sam::kNmsWord);
  B200_REQUIRE(n_keep && (n == 0 || (boxes && scores && workspace && keep)), "sam_nms: null pointer");
  B200_REQUIRE(((uintptr_t)workspace & 15) == 0, "sam_nms: workspace must be 16-byte aligned");
  cudaStream_t s = S(stream);
  if (n == 0) {
    B200_CUDA(cudaMemsetAsync(n_keep, 0, sizeof(int32_t), s));
    return 0;
  }
  Carver<16> c{static_cast<char*>(workspace)};
  int32_t* order = c.take<int32_t>(n);
  unsigned long long* mask = c.take<unsigned long long>((long long)n * words);
  sam::rank_kernel<<<ceil_div(n, 256), 256, 0, s>>>(scores, n, order);
  B200_LAUNCH_CHECK();
  sam::iou_mask_kernel<<<dim3((unsigned)ceil_div(n, 128), (unsigned)words), 128, 0, s>>>(boxes, order, n, iou_thresh,
                                                                                         mask);
  B200_LAUNCH_CHECK();
  const size_t smem = (size_t)words * 8;
  if (smem > 48 * 1024)
    B200_CUDA(cudaFuncSetAttribute(sam::greedy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  sam::greedy_kernel<<<1, 1024, smem, s>>>(mask, order, n, keep, n_keep);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_sam_mask_write(const float* logits, const int64_t* sel, int n, int lh, int lw, int grid,
                                           int in_h, int in_w, int out_h, int out_w, float thr, uint8_t* out,
                                           deva_stream_t stream) {
  sam::Shape p;
  B200_REQUIRE(sam::shape(lh, lw, grid, in_h, in_w, out_h, out_w, &p),
               "sam_mask_write: logits %d x %d, grid %d, input %d x %d, frame %d x %d out of range", lh, lw, grid, in_h,
               in_w, out_h, out_w);
  B200_REQUIRE(n >= 0 && n <= 65535, "sam_mask_write: %d masks, expected 0 to 65535", n);
  if (n == 0) return 0;
  B200_REQUIRE(logits && sel && out, "sam_mask_write: null pointer");
  const dim3 blocks((unsigned)ceil_div(out_h, sam::kBandRows), (unsigned)n);
  sam::stats_kernel<true><<<blocks, sam::kThreads, 0, S(stream)>>>(logits, sel, p, nullptr, 0.f, 0.f, 0.f, thr,
                                                                   nullptr, out);
  B200_LAUNCH_CHECK();
  return 0;
}
