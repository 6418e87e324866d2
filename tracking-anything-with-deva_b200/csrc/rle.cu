// COCO compressed RLE of every segment of an id map on the device: the counts string pycocotools.mask.encode writes
// for each mask ids == seg_ids[j] (DESIGN §7, deva/utils/rle_encode.py, oracle/coco_rle.py).  All segments come from
// one pass over the map: in column-major order, a position where the id changes is a run boundary for exactly the two
// ids involved, so only change points matter.
//   1. canon_kernel, slot_kernel: the distinct seg ids, sorted, and each entry's slot among them;
//   2. boundary_kernel<false>: one warp per chunk of column-major positions counts each slot's boundaries in it;
//   3. scan_chunks_kernel, scan_slots_kernel: per slot, the chunks' first output index; per slot, its first index in
//      the boundary list;
//   4. boundary_kernel<true>: the same walk writes each slot's boundary positions in increasing order.  A slot's
//      boundaries alternate between run starts (the new id) and run ends (the old id), so a position's rank inside a
//      32-position window follows from matching lanes of one kind and whether the slot was set before the window;
//   5. length_kernel, offsets_kernel, write_kernel: the counts are differences of boundary positions, each count (or
//      its delta from two counts before, past the third) takes 1 to 7 characters; per slot the lengths are summed, the
//      entries' offsets scanned in order, and one block per entry writes its string.
// No host synchronisation, no allocation, and the bytes depend on the inputs alone.
#include <stdint.h>

#include "common.h"
#include "scan.cuh"

namespace b200 {
namespace rle {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kWarps = 4;                  // chunks per block in the boundary passes
constexpr int kScanThreads = 1024;
constexpr int kThreads = 256;              // per-slot and per-entry kernels
constexpr long long kMinChunk = 4096;      // column-major positions per chunk (a multiple of 32)
constexpr long long kMaxCells = 1ll << 22;  // slots x chunks of per-chunk boundary counts

struct Plan {
  long long pixels, chunk;
  int chunks;
};

inline Plan plan(int h, int w, int n) {
  Plan p;
  p.pixels = (long long)h * w;
  p.chunk = kMinChunk;
  while ((long long)n * ((p.pixels + p.chunk - 1) / p.chunk) > kMaxCells) p.chunk *= 2;
  p.chunks = (int)((p.pixels + p.chunk - 1) / p.chunk);
  return p;
}

// Workspace regions, each 16-byte aligned.
struct Work {
  int* canon;           // [n] first entry with the same id
  int* entry_slot;      // [n] slot of each entry
  long long* uniq;      // [n] distinct ids, ascending (the first n_slots)
  int* n_slots;         // [1]
  int* chunk_count;     // [n * chunks] boundaries per (slot, chunk); after the scan, the chunk's first index
  int* slot_count;      // [n] boundaries per slot
  long long* slot_start;  // [n] first index of the slot's boundaries
  long long* slot_len;  // [n] characters of the slot's string
  int* bounds;          // [2 * pixels] boundary positions, grouped by slot, increasing within a slot
};

inline size_t carve(const Plan& p, int n, void* base, Work* w) {
  Carver<16> c{static_cast<char*>(base)};
  Work t;
  t.canon = c.take<int>(n);
  t.entry_slot = c.take<int>(n);
  t.uniq = c.take<long long>(n);
  t.n_slots = c.take<int>(1);
  t.chunk_count = c.take<int>((long long)n * p.chunks);
  t.slot_count = c.take<int>(n);
  t.slot_start = c.take<long long>(n);
  t.slot_len = c.take<long long>(n);
  t.bounds = c.take<int>(p.pixels * 2);
  if (w) *w = t;
  return c.bytes;
}

// ---- 1. distinct ids -----------------------------------------------------------------------------------------------
__global__ void canon_kernel(const int64_t* __restrict__ seg, int n, int* __restrict__ canon) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int64_t v = seg[j];
  int first = j;
  for (int i = 0; i < j; ++i) {
    if (seg[i] == v) {
      first = i;
      break;
    }
  }
  canon[j] = first;
}

__global__ void slot_kernel(const int64_t* __restrict__ seg, int n, const int* __restrict__ canon,
                            int* __restrict__ entry_slot, long long* __restrict__ uniq, int* __restrict__ n_slots) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int64_t v = seg[j];
  int below = 0, above = 0;
  for (int i = 0; i < n; ++i) {
    if (canon[i] != i) continue;
    const int64_t u = seg[i];
    below += u < v;
    above += u > v;
  }
  entry_slot[j] = below;
  if (canon[j] == j) {
    uniq[below] = v;
    if (above == 0) *n_slots = below + 1;
  }
}

// ---- 2, 4. boundaries ----------------------------------------------------------------------------------------------
__device__ __forceinline__ int lookup(const long long* uniq, int n_slots, long long v) {
  int lo = 0, hi = n_slots;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (uniq[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo < n_slots && uniq[lo] == v ? lo : -1;
}

// Dynamic shared memory: the n distinct ids, then one counter per slot for each warp.
template <bool kWrite>
__global__ void __launch_bounds__(32 * kWarps) boundary_kernel(const int64_t* __restrict__ ids, int h, int w, int n,
                                                               Plan p, Work wk) {
  extern __shared__ __align__(16) unsigned char smem[];
  long long* uniq = reinterpret_cast<long long*>(smem);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int* count = reinterpret_cast<int*>(smem + (size_t)n * 8) + (size_t)warp * n;
  const int n_slots = *wk.n_slots;
  for (int s = threadIdx.x; s < n_slots; s += blockDim.x) uniq[s] = wk.uniq[s];
  for (int s = lane; s < n_slots; s += 32) count[s] = 0;
  __syncthreads();
  const long long c = (long long)blockIdx.x * kWarps + warp;
  if (c >= p.chunks) return;  // whole warps leave
  const long long p0 = c * p.chunk, end = min(p0 + p.chunk, p.pixels);
  const unsigned below = (1u << lane) - 1;
  for (long long base = p0; base < end; base += 32) {
    const long long q = base + lane;
    const bool valid = q < end;
    int sa = -1, sb = -1, on = -1;
    if (valid) {
      const long long x = q / h, y = q - x * h;
      const long long cur = ids[y * w + x];
      long long prev = 0;
      if (q > 0) prev = y > 0 ? ids[(y - 1) * w + x] : ids[(long long)(h - 1) * w + x - 1];
      if (q == 0 || cur != prev) {
        sa = lookup(uniq, n_slots, cur);  // a run of cur starts at q
        if (q > 0) sb = lookup(uniq, n_slots, prev);  // a run of prev ends at q
      }
      if (kWrite && lane == 0 && q > 0) on = cur != prev ? sb : lookup(uniq, n_slots, prev);
    }
    if (!kWrite) {
      if (sa >= 0) atomicAdd(count + sa, 1);
      if (sb >= 0) atomicAdd(count + sb, 1);
      continue;
    }
    on = __shfl_sync(kFull, on, 0);  // the slot set just before the window, if any
    const unsigned ma = __match_any_sync(kFull, sa), mb = __match_any_sync(kFull, sb);
    // a slot's boundaries alternate start, end, start, ...; the first in the window is an end iff the slot was set
    if (sa >= 0) {
      const long long at = wk.slot_start[sa] + wk.chunk_count[(size_t)sa * p.chunks + c] + count[sa] +
                           2 * __popc(ma & below) + (on == sa);
      if (at < wk.slot_start[sa] + wk.slot_count[sa]) wk.bounds[at] = (int)q;
    }
    if (sb >= 0) {
      const long long at = wk.slot_start[sb] + wk.chunk_count[(size_t)sb * p.chunks + c] + count[sb] +
                           2 * __popc(mb & below) + (on != sb);
      if (at < wk.slot_start[sb] + wk.slot_count[sb]) wk.bounds[at] = (int)q;
    }
    __syncwarp();
    if (sa >= 0 && (ma & below) == 0) atomicAdd(count + sa, __popc(ma));
    if (sb >= 0 && (mb & below) == 0) atomicAdd(count + sb, __popc(mb));
    __syncwarp();
  }
  if (!kWrite) {
    __syncwarp();
    for (int s = lane; s < n_slots; s += 32) wk.chunk_count[(size_t)s * p.chunks + c] = count[s];
  }
}

// ---- 3, 5. scans ---------------------------------------------------------------------------------------------------
// One block per slot: its chunks' counts -> the chunks' first index within the slot; the slot's total.
__global__ void __launch_bounds__(kScanThreads) scan_chunks_kernel(Plan p, Work wk) {
  __shared__ long long warp_sums[kScanThreads / 32];
  const int s = blockIdx.x;
  if (s >= *wk.n_slots) return;
  int* row = wk.chunk_count + (size_t)s * p.chunks;
  const long long total = block_scan(
      p.chunks, 0ll, warp_sums, [&](long long k) { return row[k]; },
      [&](long long k, long long o, int) { row[k] = (int)o; });
  if (threadIdx.x == 0) wk.slot_count[s] = (int)total;
}

__global__ void __launch_bounds__(kScanThreads) scan_slots_kernel(Work wk) {
  __shared__ long long warp_sums[kScanThreads / 32];
  block_scan(
      *wk.n_slots, 0ll, warp_sums, [&](long long s) { return wk.slot_count[s]; },
      [&](long long s, long long o, int) { wk.slot_start[s] = o; });
}

// ---- 5. strings ----------------------------------------------------------------------------------------------------
// Count i of a slot with k boundaries at b[0..k): b[0] - 0, b[i] - b[i - 1], ..., pixels - b[k - 1].
__device__ __forceinline__ long long run(const int* b, int k, long long pixels, long long i) {
  const long long hi = i == k ? pixels : b[i];
  const long long lo = i == 0 ? 0 : b[i - 1];
  return hi - lo;
}

// The value rleToString codes for count i: the count, less the count two before when i > 2.
__device__ __forceinline__ long long coded(const int* b, int k, long long pixels, long long i) {
  return run(b, k, pixels, i) - (i > 2 ? run(b, k, pixels, i - 2) : 0);
}

__device__ __forceinline__ int chars(long long x) {
  int n = 1;
  for (;;) {
    const int c = (int)(x & 0x1f);
    x >>= 5;
    if (!((c & 0x10) ? x != -1 : x != 0)) return n;
    ++n;
  }
}

__device__ __forceinline__ void emit(long long x, uint8_t* out, long long at, long long end) {
  for (;;) {
    int c = (int)(x & 0x1f);
    x >>= 5;
    const bool more = (c & 0x10) ? x != -1 : x != 0;
    if (more) c |= 0x20;
    if (at < end) out[at] = (uint8_t)(48 + c);
    ++at;
    if (!more) return;
  }
}

// One block per slot: the length of its string.
__global__ void __launch_bounds__(kThreads) length_kernel(long long pixels, Work wk) {
  __shared__ long long warp_sums[kThreads / 32];
  const int s = blockIdx.x;
  if (s >= *wk.n_slots) return;
  const int k = wk.slot_count[s];
  const int* b = wk.bounds + wk.slot_start[s];
  long long len = 0;
  for (long long i = threadIdx.x; i <= k; i += kThreads) len += chars(coded(b, k, pixels, i));
  long long total;
  block_exclusive_scan(len, warp_sums, total);
  if (threadIdx.x == 0) wk.slot_len[s] = total;
}

__global__ void __launch_bounds__(kScanThreads) offsets_kernel(int n, Work wk, int64_t* __restrict__ offsets) {
  __shared__ long long warp_sums[kScanThreads / 32];
  const long long total = block_scan(
      n, 0ll, warp_sums, [&](long long j) { return wk.slot_len[wk.entry_slot[j]]; },
      [&](long long j, long long o, long long) { offsets[j] = o; });
  if (threadIdx.x == 0) offsets[n] = total;
}

// One block per entry: its slot's string at offsets[j].
__global__ void __launch_bounds__(kThreads) write_kernel(long long pixels, Work wk, const int64_t* __restrict__ offsets,
                                                         uint8_t* __restrict__ out) {
  __shared__ long long warp_sums[kThreads / 32];
  const int j = blockIdx.x;
  const int s = wk.entry_slot[j];
  const int k = wk.slot_count[s];
  const int* b = wk.bounds + wk.slot_start[s];
  const long long end = offsets[j + 1];
  long long x = 0;  // the coded value the thread loaded last, written once its offset is known
  block_scan(
      k + 1ll, (long long)offsets[j], warp_sums,
      [&](long long i) {
        x = coded(b, k, pixels, i);
        return chars(x);
      },
      [&](long long, long long at, int) { emit(x, out, at, end); });
}

}  // namespace rle
}  // namespace b200

using namespace b200;

extern "C" {

DEVA_B200_API size_t deva_b200_rle_bound(int h, int w, int n) {
  if (h < 1 || w < 1 || n < 1) return 0;
  // A coded value's chunks beyond the first are charged to the larger of the two counts it involves, so a count c >= 1
  // carries at most 1 + 2 E(c) <= c characters (E(c): c's own chunks beyond the first) and a leading 0 one.  A string
  // is at most pixels + 1 characters, reached when the mask changes at every pixel.
  return (size_t)n * (size_t)((long long)h * w + 1);
}

DEVA_B200_API size_t deva_b200_rle_workspace_bytes(int h, int w, int n) {
  if (h < 1 || w < 1 || n < 1) return 0;
  return rle::carve(rle::plan(h, w, n), n, nullptr, nullptr);
}

DEVA_B200_API int deva_b200_rle_encode(const int64_t* ids, int h, int w, const int64_t* seg_ids, int n, void* workspace,
                                       uint8_t* out, int64_t* offsets, deva_stream_t stream) {
  B200_REQUIRE(ids && seg_ids && workspace && out && offsets, "rle_encode: null pointer");
  B200_REQUIRE(h >= 1 && w >= 1 && (long long)h * w < (1ll << 31),
               "rle_encode: %d x %d map, expected 1 <= h, w and h * w < 2^31", h, w);
  B200_REQUIRE(n >= 1 && n <= DEVA_B200_MAX_SEGMENT_CHANNELS, "rle_encode: %d seg ids, expected 1 to %d", n,
               DEVA_B200_MAX_SEGMENT_CHANNELS);
  B200_REQUIRE(((uintptr_t)ids & 7) == 0 && ((uintptr_t)seg_ids & 7) == 0 && ((uintptr_t)offsets & 7) == 0 &&
                   ((uintptr_t)workspace & 15) == 0,
               "rle_encode: ids, seg_ids and offsets must be 8-byte and workspace 16-byte aligned");
  const rle::Plan p = rle::plan(h, w, n);
  rle::Work wk;
  rle::carve(p, n, workspace, &wk);
  cudaStream_t s = S(stream);
  const unsigned entry_blocks = (unsigned)ceil_div(n, rle::kThreads);
  rle::canon_kernel<<<entry_blocks, rle::kThreads, 0, s>>>(seg_ids, n, wk.canon);
  B200_LAUNCH_CHECK();
  rle::slot_kernel<<<entry_blocks, rle::kThreads, 0, s>>>(seg_ids, n, wk.canon, wk.entry_slot, wk.uniq, wk.n_slots);
  B200_LAUNCH_CHECK();
  const size_t smem = (size_t)n * 8 + (size_t)rle::kWarps * n * 4;
  if (smem > 48 * 1024) {
    B200_CUDA(cudaFuncSetAttribute(rle::boundary_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    B200_CUDA(cudaFuncSetAttribute(rle::boundary_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  const unsigned chunk_blocks = (unsigned)ceil_div(p.chunks, rle::kWarps);
  rle::boundary_kernel<false><<<chunk_blocks, 32 * rle::kWarps, smem, s>>>(ids, h, w, n, p, wk);
  B200_LAUNCH_CHECK();
  rle::scan_chunks_kernel<<<n, rle::kScanThreads, 0, s>>>(p, wk);
  B200_LAUNCH_CHECK();
  rle::scan_slots_kernel<<<1, rle::kScanThreads, 0, s>>>(wk);
  B200_LAUNCH_CHECK();
  rle::boundary_kernel<true><<<chunk_blocks, 32 * rle::kWarps, smem, s>>>(ids, h, w, n, p, wk);
  B200_LAUNCH_CHECK();
  rle::length_kernel<<<n, rle::kThreads, 0, s>>>(p.pixels, wk);
  B200_LAUNCH_CHECK();
  rle::offsets_kernel<<<1, rle::kScanThreads, 0, s>>>(n, wk, offsets);
  B200_LAUNCH_CHECK();
  rle::write_kernel<<<n, rle::kThreads, 0, s>>>(p.pixels, wk, offsets, out);
  B200_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
