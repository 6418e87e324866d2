// Block-wide exclusive scans and workspace carving shared by the device encoders (png.cu, jpeg.cu, rle.cu).
#pragma once
#include <stddef.h>

namespace b200 {

// Exclusive scan of one value per thread over the block (blockDim.x a multiple of 32, at most 1024; warp_sums holds
// one value per warp).  Returns the thread's offset and sets total to the block's sum.  The trailing barrier lets the
// caller reuse warp_sums at once.
template <typename T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* warp_sums, T& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  T x = v;  // inclusive scan within the warp
  for (int m = 1; m < 32; m <<= 1) {
    const T t = __shfl_up_sync(0xffffffffu, x, m);
    if (lane >= m) x += t;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  T before = 0;
  total = 0;
  for (int k = 0; k < warps; ++k) {
    if (k < warp) before += warp_sums[k];
    total += warp_sums[k];
  }
  __syncthreads();  // warp_sums is rewritten by the next call
  return before + x - v;
}

// Exclusive scan of n values by one block, blockDim.x * kItems values per chunk and kItems consecutive values per
// thread: load(i) is value i, store(i, offset, value) receives its offset, counted from carry.  Returns carry plus the
// values' sum on every thread.  Each thread loads and stores only its own values, so the scan may run in place.
template <int kItems = 1, typename T, typename Load, typename Store>
__device__ __forceinline__ T block_scan(long long n, T carry, T* warp_sums, Load load, Store store) {
  using V = decltype(load(0ll));
  for (long long base = 0; base < n; base += (long long)blockDim.x * kItems) {
    const long long i0 = base + (long long)threadIdx.x * kItems;
    V v[kItems];
    T sum = 0;
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      v[k] = i0 + k < n ? load(i0 + k) : V(0);
      sum += v[k];
    }
    T chunk;
    T o = carry + block_exclusive_scan(sum, warp_sums, chunk);
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      if (i0 + k < n) store(i0 + k, o, v[k]);
      o += v[k];
    }
    carry += chunk;
  }
  return carry;
}

// Lays out a workspace region by region, each starting kAlign-aligned: take<T>(count) returns the next region and
// `bytes` is the size so far.  On a null base the regions are null and only `bytes` counts, so the one layout both
// sizes a workspace and carves it.
template <size_t kAlign>
struct Carver {
  char* base;
  size_t bytes = 0;

  template <typename T>
  __host__ __device__ T* take(long long count) {
    T* at = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += ((size_t)count * sizeof(T) + kAlign - 1) / kAlign * kAlign;
    return at;
  }
};

}  // namespace b200
