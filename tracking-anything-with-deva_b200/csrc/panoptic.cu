// Video panoptic metrics on the device (deva/vps_metrics): the joint label histogram of a ground-truth and a predicted
// RGB id frame, and the id remap of stuff merging.  Both decode id = r + 256 g + 65536 b per pixel and map it to its index
// in a sorted id table by binary search in shared memory; an id that is not in the table maps to the index n_table.
// Counts are warp-aggregated (__match_any_sync) before the atomic, since most neighbouring pixels share one label.
#include <algorithm>
#include <stdint.h>

#include "common.h"

namespace b200 {
namespace pano {

constexpr int kThreads = 1024;
constexpr int kPixelsPerThread = 4;  // 4 RGB pixels = 3 aligned 32-bit words
// Shared memory a histogram may take before the joint histogram falls back to global atomics (the tables come on top).
constexpr size_t kMaxSmemBytes = 200 * 1024;

// index of v in the sorted table t[0, n), or n
__device__ __forceinline__ int table_index(const int* __restrict__ t, int n, int v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (t[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return (lo < n && t[lo] == v) ? lo : n;
}

// The ids of pixels 4q .. 4q+3 of an RGB u8 frame (all four in range): three 32-bit loads when the frame is 4-byte aligned.
__device__ __forceinline__ void load4(const uint8_t* __restrict__ rgb, long long q, bool aligned, int (&id)[4]) {
  uint8_t b[12];
  if (aligned) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(rgb) + 3 * q;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const uint32_t v = __ldg(w + k);
#pragma unroll
      for (int j = 0; j < 4; ++j) b[4 * k + j] = (uint8_t)(v >> (8 * j));
    }
  } else {
#pragma unroll
    for (int k = 0; k < 12; ++k) b[k] = __ldg(rgb + 12 * q + k);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) id[j] = b[3 * j] | (b[3 * j + 1] << 8) | (b[3 * j + 2] << 16);
}

__device__ __forceinline__ int load1(const uint8_t* __restrict__ rgb, long long i) {
  return __ldg(rgb + 3 * i) | (__ldg(rgb + 3 * i + 1) << 8) | (__ldg(rgb + 3 * i + 2) << 16);
}

// One add per distinct cell among the warp's active lanes.
template <typename T>
__device__ __forceinline__ void warp_add(T* hist, int cell, unsigned active) {
  const unsigned peers = __match_any_sync(active, cell);
  if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(hist + cell, (T)__popc(peers));
}

// hist[(n_gt + 1) x (n_pred + 1)] += joint counts of (gt index, pred index).  kShared: a block-private histogram in
// shared memory, merged into `hist` (non-zero cells only) at the end; otherwise every add goes to global memory.
template <bool kShared>
__global__ void __launch_bounds__(kThreads)
joint_hist_kernel(const uint8_t* __restrict__ gt, const uint8_t* __restrict__ pred, long long n_pix,
                  const int* __restrict__ gt_ids, int n_gt, const int* __restrict__ pred_ids, int n_pred,
                  int* __restrict__ hist) {
  extern __shared__ int smem[];
  int* s_gt = smem;
  int* s_pred = s_gt + n_gt;
  int* s_hist = s_pred + n_pred;
  const int cols = n_pred + 1;
  const int cells = (n_gt + 1) * cols;
  for (int k = threadIdx.x; k < n_gt; k += kThreads) s_gt[k] = gt_ids[k];
  for (int k = threadIdx.x; k < n_pred; k += kThreads) s_pred[k] = pred_ids[k];
  if (kShared)
    for (int k = threadIdx.x; k < cells; k += kThreads) s_hist[k] = 0;
  __syncthreads();
  int* h = kShared ? s_hist : hist;

  const bool aligned = ((reinterpret_cast<uintptr_t>(gt) | reinterpret_cast<uintptr_t>(pred)) & 3) == 0;
  const long long n_quads = n_pix / kPixelsPerThread;
  const long long n_iter = (n_quads + kThreads - 1) / kThreads;  // whole warps iterate together (the match needs it)
  int last_g = -1, last_gi = 0, last_p = -1, last_pi = 0;
  for (long long it = blockIdx.x; it < n_iter; it += gridDim.x) {
    const long long q = it * kThreads + threadIdx.x;
    const bool live = q < n_quads;
    const unsigned active = __ballot_sync(0xffffffffu, live);
    if (!live) continue;
    int g[4], p[4];
    load4(gt, q, aligned, g);
    load4(pred, q, aligned, p);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (g[j] != last_g) { last_g = g[j]; last_gi = table_index(s_gt, n_gt, g[j]); }
      if (p[j] != last_p) { last_p = p[j]; last_pi = table_index(s_pred, n_pred, p[j]); }
      warp_add(h, last_gi * cols + last_pi, active);
    }
  }
  // the n_pix % 4 trailing pixels
  if (blockIdx.x == 0 && threadIdx.x < n_pix - n_quads * kPixelsPerThread) {
    const long long i = n_quads * kPixelsPerThread + threadIdx.x;
    const int gi = table_index(s_gt, n_gt, load1(gt, i)), pi = table_index(s_pred, n_pred, load1(pred, i));
    atomicAdd(h + gi * cols + pi, 1);
  }
  if (kShared) {
    __syncthreads();
    for (int k = threadIdx.x; k < cells; k += kThreads)
      if (s_hist[k]) atomicAdd(hist + k, s_hist[k]);
  }
}

// Stuff merging's remap: out id = out_ids[slot[index of the pred id]], written as RGB bytes (id >> 8i) & 255; counts[s]
// = pixels written with out_ids[s]; *unknown = pixels whose id is not in the table (they take slot[n_table]).
__global__ void __launch_bounds__(kThreads)
remap_kernel(const uint8_t* __restrict__ pred, long long n_pix, const int* __restrict__ ids, int n_table,
             const int* __restrict__ slot, const int* __restrict__ out_ids, int n_out, uint8_t* __restrict__ out,
             int* __restrict__ counts, int* __restrict__ unknown) {
  extern __shared__ int smem[];
  int* s_ids = smem;                 // [n_table]
  int* s_slot = s_ids + n_table;     // [n_table + 1]
  int* s_out = s_slot + n_table + 1; // [n_out]
  int* s_cnt = s_out + n_out;        // [n_out + 1]: the last one counts unknown ids
  for (int k = threadIdx.x; k < n_table; k += kThreads) s_ids[k] = ids[k];
  for (int k = threadIdx.x; k <= n_table; k += kThreads) s_slot[k] = slot[k];
  for (int k = threadIdx.x; k < n_out; k += kThreads) s_out[k] = out_ids[k];
  for (int k = threadIdx.x; k <= n_out; k += kThreads) s_cnt[k] = 0;
  __syncthreads();
  const long long n_iter = (n_pix + kThreads - 1) / kThreads;
  int last = -1, last_i = 0;
  for (long long it = blockIdx.x; it < n_iter; it += gridDim.x) {
    const long long i = it * kThreads + threadIdx.x;
    const bool live = i < n_pix;
    const unsigned active = __ballot_sync(0xffffffffu, live);
    if (!live) continue;
    const int v = load1(pred, i);
    if (v != last) { last = v; last_i = table_index(s_ids, n_table, v); }
    const int s = s_slot[last_i];
    const int o = s_out[s];
    out[3 * i] = (uint8_t)(o & 255);
    out[3 * i + 1] = (uint8_t)((o >> 8) & 255);
    out[3 * i + 2] = (uint8_t)((o >> 16) & 255);
    warp_add(s_cnt, s, active);
    const unsigned unk = __ballot_sync(active, last_i == n_table);
    if (unk && (threadIdx.x & 31) == __ffs(unk) - 1) atomicAdd(s_cnt + n_out, __popc(unk));
  }
  __syncthreads();
  for (int k = threadIdx.x; k < n_out; k += kThreads)
    if (s_cnt[k]) atomicAdd(counts + k, s_cnt[k]);
  if (threadIdx.x == 0 && s_cnt[n_out]) atomicAdd(unknown, s_cnt[n_out]);
}

}  // namespace pano
}  // namespace b200

using namespace b200;

extern "C" {

DEVA_B200_API int deva_b200_pano_joint_hist(const uint8_t* gt, const uint8_t* pred, int h, int w, const int32_t* gt_ids,
                                            int n_gt, const int32_t* pred_ids, int n_pred, int32_t* hist,
                                            deva_stream_t stream) {
  B200_REQUIRE(gt && pred && hist && h > 0 && w > 0 && n_gt >= 0 && n_pred >= 0 && (gt_ids || !n_gt) &&
                   (pred_ids || !n_pred),
               "pano_joint_hist: bad arguments");
  const long long cells = (long long)(n_gt + 1) * (n_pred + 1);
  B200_REQUIRE(cells < (1ll << 31), "pano_joint_hist: %lld cells, at most 2^31 - 1", cells);
  const size_t table_bytes = (size_t)(n_gt + n_pred) * sizeof(int);
  const size_t hist_bytes = (size_t)cells * sizeof(int);
  B200_REQUIRE(table_bytes <= pano::kMaxSmemBytes, "pano_joint_hist: %d + %d ids do not fit in shared memory", n_gt,
               n_pred);
  const bool shared = table_bytes + hist_bytes <= pano::kMaxSmemBytes;
  const cudaStream_t s = S(stream);
  B200_CUDA(cudaMemsetAsync(hist, 0, hist_bytes, s));
  const long long n_pix = (long long)h * w;
  const long long quads = (n_pix / pano::kPixelsPerThread + pano::kThreads - 1) / pano::kThreads;
  const size_t smem = table_bytes + (shared ? hist_bytes : 0);
  // one block per SM at most: a shared histogram costs a zeroing and a merge pass per block
  const long long blocks = std::min<long long>(std::max(quads, 1ll), sm_count());
  if (shared) {
    B200_CUDA(cudaFuncSetAttribute(pano::joint_hist_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)smem));
    pano::joint_hist_kernel<true><<<(unsigned)blocks, pano::kThreads, smem, s>>>(gt, pred, n_pix, gt_ids, n_gt,
                                                                                 pred_ids, n_pred, hist);
  } else {
    B200_CUDA(cudaFuncSetAttribute(pano::joint_hist_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)smem));
    pano::joint_hist_kernel<false><<<(unsigned)blocks, pano::kThreads, smem, s>>>(gt, pred, n_pix, gt_ids, n_gt,
                                                                                  pred_ids, n_pred, hist);
  }
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_pano_remap(const uint8_t* pred, int h, int w, const int32_t* ids, int n_table,
                                       const int32_t* slot, const int32_t* out_ids, int n_out, uint8_t* out,
                                       int32_t* counts, int32_t* unknown, deva_stream_t stream) {
  B200_REQUIRE(pred && slot && out_ids && out && counts && unknown && h > 0 && w > 0 && n_table >= 0 && n_out >= 1 &&
                   (ids || !n_table),
               "pano_remap: bad arguments");
  const size_t smem = (size_t)(2 * n_table + 2 * n_out + 2) * sizeof(int);
  B200_REQUIRE(smem <= pano::kMaxSmemBytes, "pano_remap: %d ids and %d output ids do not fit in shared memory", n_table,
               n_out);
  const cudaStream_t s = S(stream);
  B200_CUDA(cudaMemsetAsync(counts, 0, (size_t)n_out * sizeof(int32_t), s));
  B200_CUDA(cudaMemsetAsync(unknown, 0, sizeof(int32_t), s));
  const long long n_pix = (long long)h * w;
  const long long blocks = std::max(1ll, std::min<long long>((n_pix + pano::kThreads - 1) / pano::kThreads, sm_count()));
  B200_CUDA(cudaFuncSetAttribute(pano::remap_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  pano::remap_kernel<<<(unsigned)blocks, pano::kThreads, smem, s>>>(pred, n_pix, ids, n_table, slot, out_ids, n_out, out,
                                                                    counts, unknown);
  B200_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
