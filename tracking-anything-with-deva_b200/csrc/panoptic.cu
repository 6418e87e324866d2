// Video panoptic metrics on the device (deva/vps_metrics): the joint label histogram of a ground-truth and a predicted
// RGB id frame, and the id remap of stuff merging.  Both decode id = r + 256 g + 65536 b per pixel and map it to its index
// in a sorted id table by binary search in shared memory; an id that is not in the table maps to the index n_table.
// Counts are warp-aggregated (__match_any_sync) before the atomic, since most neighbouring pixels share one label.
// The label kernels below (per-frame label areas and a label -> index rewrite) serve the unsupervised DAVIS 2017
// post-processing in the same way.
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

// Label statistics and rewrite of one decoded index or colour frame (deva/inference/postprocess_unsup_davis17.py).  A
// 1-channel frame's label is its byte; a 3- or 4-channel frame's is r << 16 | g << 8 | b (alpha ignored).  Label 0 is
// background.
namespace label_ops {

constexpr int kThreads = 1024;
constexpr int kLog2Slots = 12;
constexpr int kSharedSlots = 1 << kLog2Slots;  // block-private hash table of a colour frame: 32 KiB of keys and counts
constexpr int kSharedProbes = 32;             // a label that finds no slot within this many goes to the global table

// The labels of pixels 4q .. 4q+3 (all four in range): C 32-bit loads when the frame is 4-byte aligned.
template <int C>
__device__ __forceinline__ void load4(const uint8_t* __restrict__ f, long long q, bool aligned, int (&v)[4]) {
  uint8_t b[4 * C];
  if (aligned) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(f) + C * q;
#pragma unroll
    for (int k = 0; k < C; ++k) {
      const uint32_t x = __ldg(w + k);
#pragma unroll
      for (int j = 0; j < 4; ++j) b[4 * k + j] = (uint8_t)(x >> (8 * j));
    }
  } else {
#pragma unroll
    for (int k = 0; k < 4 * C; ++k) b[k] = __ldg(f + 4 * C * q + k);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = C == 1 ? b[j] : (b[C * j] << 16) | (b[C * j + 1] << 8) | b[C * j + 2];
}

template <int C>
__device__ __forceinline__ int load1(const uint8_t* __restrict__ f, long long i) {
  return C == 1 ? __ldg(f + i) : (__ldg(f + C * i) << 16) | (__ldg(f + C * i + 1) << 8) | __ldg(f + C * i + 2);
}

__device__ __forceinline__ unsigned mix(int v) { return (unsigned)v * 2654435761u; }

// counts[slot of label] += n in an open-addressed table (key 0 = empty slot, linear probing over at most `probes`
// slots from the label's home slot); false when none of them is free or holds the label.
__device__ __forceinline__ bool table_add(int* keys, int* counts, unsigned cap, unsigned home, int probes, int label,
                                          int n) {
  unsigned s = home;
  for (int p = 0; p < probes; ++p) {
    int k = *(volatile int*)(keys + s);
    if (k == 0) k = atomicCAS(keys + s, 0, label);
    if (k == 0 || k == label) {
      atomicAdd(counts + s, n);
      return true;
    }
    if (++s == cap) s = 0;
  }
  return false;
}

// Pixel counts of the non-zero labels.  Each block counts its pixels into shared memory (a 256-bin histogram for one
// channel, a hash table for colour; pixels of equal label in a warp are one add) and merges the non-zero entries into
// the global table keys / counts [cap]; a colour label that finds no shared slot goes to the global table directly.  The
// last block to finish compacts the global table in place into its first n entries and writes state[0] = n, or leaves
// state[0] = -1 when some label found no global slot.  state[1] counts finished blocks.
template <int C>
__global__ void __launch_bounds__(kThreads)
areas_kernel(const uint8_t* __restrict__ f, long long n_pix, int cap, int* keys, int* counts, int* state) {
  constexpr int kSlots = C == 1 ? 256 : kSharedSlots;
  __shared__ int s_keys[C == 1 ? 1 : kSlots];
  __shared__ int s_cnt[kSlots];
  __shared__ int s_warp[kThreads / 32];
  __shared__ bool s_last;
  for (int k = threadIdx.x; k < kSlots; k += kThreads) {
    s_cnt[k] = 0;
    if (C != 1) s_keys[k] = 0;
  }
  __syncthreads();
  const unsigned lane = threadIdx.x & 31;
  bool lost = false;  // some label found no global slot
  auto add = [&](int v, int n) {
    if (C == 1) {
      atomicAdd(s_cnt + v, n);
    } else if (!table_add(s_keys, s_cnt, kSlots, mix(v) >> (32 - kLog2Slots), kSharedProbes, v, n)) {
      lost |= !table_add(keys, counts, cap, mix(v) % (unsigned)cap, cap, v, n);
    }
  };

  const bool aligned = (reinterpret_cast<uintptr_t>(f) & 3) == 0;
  const long long n_quads = n_pix / 4;
  const long long n_iter = (n_quads + kThreads - 1) / kThreads;  // whole warps iterate together (the match needs it)
  for (long long it = blockIdx.x; it < n_iter; it += gridDim.x) {
    const long long q = it * kThreads + threadIdx.x;
    const bool live = q < n_quads;
    const unsigned active = __ballot_sync(0xffffffffu, live);
    if (!live) continue;
    int v[4];
    load4<C>(f, q, aligned, v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const unsigned peers = __match_any_sync(active, v[j]);
      if (v[j] != 0 && lane == __ffs(peers) - 1) add(v[j], __popc(peers));
    }
  }
  // the n_pix % 4 trailing pixels
  if (blockIdx.x == 0 && threadIdx.x < n_pix - n_quads * 4) {
    const int v = load1<C>(f, n_quads * 4 + threadIdx.x);
    if (v != 0) add(v, 1);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < kSlots; k += kThreads) {
    const int n = s_cnt[k], v = C == 1 ? k : s_keys[k];
    if (n != 0 && v != 0) lost |= !table_add(keys, counts, cap, mix(v) % (unsigned)cap, cap, v, n);
  }
  if (lost) atomicExch(state, -1);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(state + 1, 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (__ldcg(state) < 0) return;
  // in-place compaction, one chunk of kThreads slots at a time: every slot of a chunk is read before any is written, and
  // an entry only moves to a lower index
  const unsigned warp = threadIdx.x >> 5;
  int total = 0;
  for (int base = 0; base < cap; base += kThreads) {
    const int k = base + threadIdx.x;
    const int key = k < cap ? __ldcg(keys + k) : 0;
    const int cnt = k < cap ? __ldcg(counts + k) : 0;
    const unsigned kept = __ballot_sync(0xffffffffu, key != 0);
    if (lane == 0) s_warp[warp] = __popc(kept);
    __syncthreads();
    int before = 0, chunk = 0;
    for (int i = 0; i < kThreads / 32; ++i) {
      const int c = s_warp[i];
      before += i < (int)warp ? c : 0;
      chunk += c;
    }
    if (key != 0) {
      const int pos = total + before + __popc(kept & ((1u << lane) - 1));
      keys[pos] = key;
      counts[pos] = cnt;
    }
    total += chunk;
    __syncthreads();
  }
  if (threadIdx.x == 0) state[0] = total;
}

// out[pixel] = index[i] where labels[i] is the pixel's label (labels sorted ascending, n entries), else 0.
template <int C>
__global__ void __launch_bounds__(kThreads)
index_kernel(const uint8_t* __restrict__ f, long long n_pix, const int* __restrict__ labels,
             const int* __restrict__ index, int n, uint8_t* __restrict__ out) {
  extern __shared__ int smem[];
  int* s_lab = smem;
  int* s_idx = smem + n;
  for (int k = threadIdx.x; k < n; k += kThreads) {
    s_lab[k] = labels[k];
    s_idx[k] = index[k];
  }
  __syncthreads();
  auto lookup = [&](int v) {
    const int i = pano::table_index(s_lab, n, v);
    return i < n ? s_idx[i] : 0;
  };
  const bool aligned = ((reinterpret_cast<uintptr_t>(f) | reinterpret_cast<uintptr_t>(out)) & 3) == 0;
  const long long n_quads = n_pix / 4;
  int last = -1, last_o = 0;
  for (long long q = (long long)blockIdx.x * kThreads + threadIdx.x; q < n_quads; q += (long long)gridDim.x * kThreads) {
    int v[4];
    load4<C>(f, q, aligned, v);
    uint32_t word = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (v[j] != last) {
        last = v[j];
        last_o = lookup(v[j]);
      }
      word |= (uint32_t)(last_o & 255) << (8 * j);
    }
    if (aligned) {
      reinterpret_cast<uint32_t*>(out)[q] = word;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) out[4 * q + j] = (uint8_t)(word >> (8 * j));
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < n_pix - n_quads * 4) {
    const long long i = n_quads * 4 + threadIdx.x;
    out[i] = (uint8_t)lookup(load1<C>(f, i));
  }
}

}  // namespace label_ops
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

DEVA_B200_API int deva_b200_label_areas(const uint8_t* frame, int h, int w, int channels, int capacity, int32_t* labels,
                                        int32_t* counts, int32_t* state, deva_stream_t stream) {
  B200_REQUIRE(frame && labels && counts && state && h > 0 && w > 0 && capacity > 0, "label_areas: bad arguments");
  B200_REQUIRE(channels == 1 || channels == 3 || channels == 4, "label_areas: %d channels, expected 1, 3 or 4",
               channels);
  const cudaStream_t s = S(stream);
  B200_CUDA(cudaMemsetAsync(labels, 0, (size_t)capacity * sizeof(int32_t), s));
  B200_CUDA(cudaMemsetAsync(counts, 0, (size_t)capacity * sizeof(int32_t), s));
  B200_CUDA(cudaMemsetAsync(state, 0, 2 * sizeof(int32_t), s));
  const long long n_pix = (long long)h * w;
  // a block clears and merges a whole shared table, so it should count a few rounds of pixels first
  const long long rounds = (n_pix / 4 + label_ops::kThreads - 1) / label_ops::kThreads;
  const unsigned blocks = (unsigned)std::max(1ll, std::min<long long>((rounds + 3) / 4, sm_count()));
  if (channels == 1)
    label_ops::areas_kernel<1><<<blocks, label_ops::kThreads, 0, s>>>(frame, n_pix, capacity, labels, counts, state);
  else if (channels == 3)
    label_ops::areas_kernel<3><<<blocks, label_ops::kThreads, 0, s>>>(frame, n_pix, capacity, labels, counts, state);
  else
    label_ops::areas_kernel<4><<<blocks, label_ops::kThreads, 0, s>>>(frame, n_pix, capacity, labels, counts, state);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_label_to_index(const uint8_t* frame, int h, int w, int channels, const int32_t* labels,
                                           const int32_t* index, int n, uint8_t* out, deva_stream_t stream) {
  B200_REQUIRE(frame && out && h > 0 && w > 0 && n >= 0 && (n == 0 || (labels && index)),
               "label_to_index: bad arguments");
  B200_REQUIRE(channels == 1 || channels == 3 || channels == 4, "label_to_index: %d channels, expected 1, 3 or 4",
               channels);
  const size_t smem = (size_t)2 * n * sizeof(int);
  B200_REQUIRE(smem <= pano::kMaxSmemBytes, "label_to_index: %d labels do not fit in shared memory", n);
  const cudaStream_t s = S(stream);
  const long long n_pix = (long long)h * w;
  const unsigned blocks = (unsigned)std::max(
      1ll, std::min<long long>((n_pix / 4 + label_ops::kThreads - 1) / label_ops::kThreads, 2ll * sm_count()));
  if (channels == 1) {
    B200_CUDA(cudaFuncSetAttribute(label_ops::index_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    label_ops::index_kernel<1><<<blocks, label_ops::kThreads, smem, s>>>(frame, n_pix, labels, index, n, out);
  } else if (channels == 3) {
    B200_CUDA(cudaFuncSetAttribute(label_ops::index_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    label_ops::index_kernel<3><<<blocks, label_ops::kThreads, smem, s>>>(frame, n_pix, labels, index, n, out);
  } else {
    B200_CUDA(cudaFuncSetAttribute(label_ops::index_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    label_ops::index_kernel<4><<<blocks, label_ops::kThreads, smem, s>>>(frame, n_pix, labels, index, n, out);
  }
  B200_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
