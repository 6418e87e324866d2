// PNG image data decoded on the device (deva/utils/png_decode.py; the format rules are DESIGN §7): a batch of files'
// zlib streams -> Pillow's arrays.  The host has parsed the chunks and decided each file is device-eligible; here every
// stream is checked as it is decoded, and a file whose status is nonzero is left to Pillow.
//   1. inflate_kernel: one warp per file.  Lane 0 decodes the symbols (inflate.cuh) into the file's filtered stream in
//      the workspace, keeping the last 64 KiB in shared memory, where matches read their source; every match of at
//      least kWarpCopy bytes is copied by the whole warp.  Then the warp forms the Adler-32 from per-lane partial sums
//      and compares it with the trailer.
//   2. unfilter_kernel: one block per file, a wavefront over bands of rows: thread t owns row band + t and at step s
//      reconstructs its pixel s - t, so a pixel's left, upper and upper-left neighbours are done one step or more
//      before it, with one barrier per step.  The same pass checks the filter types, unpacks sub-byte rows MSB-first,
//      scales 2- and 4-bit grey by 85 and 17 and writes Pillow's layout ([h, w] or [h, w, 3 | 4]).
#include <stdint.h>

#include "common.h"
#include "inflate.cuh"
#include "scan.cuh"

namespace b200 {
namespace png_decode {

using namespace inflate;

constexpr unsigned kFull = 0xffffffffu;
constexpr int kWarpCopy = 16;  // shorter matches are copied by lane 0 as it decodes
constexpr int kUnfilterThreads = 1024;

// One file's descriptor: int64 [kDescFields] (include/deva_b200.h).
enum Field { kStreamOff, kStreamLen, kH, kW, kColourType, kBits, kOutOff, kWorkOff, kDescFields };

struct Shape {
  long long h, w;
  int channels, bits;
  long long rowbytes;  // packed bytes of a row, without its filter byte
  int bpp;             // bytes per complete pixel, at least 1
  __host__ __device__ long long filtered() const { return h * (rowbytes + 1); }
};

// The shape of a supported (colour type, bit depth): grey 2, 4, 8; palette 1, 2, 4, 8; RGB 8; RGBA 8.
__host__ __device__ inline bool shape_of(long long h, long long w, long long colour_type, long long bits, Shape* g) {
  const bool ok = h >= 1 && w >= 1 && h <= (1 << 30) && w <= (1 << 30) &&
                  ((colour_type == 0 && (bits == 2 || bits == 4 || bits == 8)) ||
                   (colour_type == 3 && (bits == 1 || bits == 2 || bits == 4 || bits == 8)) ||
                   ((colour_type == 2 || colour_type == 6) && bits == 8));
  if (!ok) return false;
  const int channels = colour_type == 2 ? 3 : colour_type == 6 ? 4 : 1;
  *g = Shape{h, w, channels, (int)bits, (w * channels * bits + 7) / 8, (int)(channels * bits / 8 > 1 ? channels * bits / 8 : 1)};
  return true;
}

constexpr size_t kInflateSmem = sizeof(Tables) + kWindow;

__global__ void __launch_bounds__(32) inflate_kernel(const uint8_t* __restrict__ streams,
                                                     const int64_t* __restrict__ desc, int n,
                                                     uint8_t* __restrict__ work, int* __restrict__ status) {
  extern __shared__ __align__(16) uint8_t smem[];
  Tables& tables = *reinterpret_cast<Tables*>(smem);
  uint8_t* window = smem + sizeof(Tables);
  const int f = blockIdx.x, lane = threadIdx.x;
  if (f >= n) return;
  const int64_t* d = desc + (size_t)f * kDescFields;
  Shape g;
  if (!shape_of(d[kH], d[kW], d[kColourType], d[kBits], &g) || d[kStreamOff] < 0 || d[kStreamLen] < 0 ||
      d[kOutOff] < 0 || d[kWorkOff] < 0) {
    if (lane == 0) status[f] = kBadDescriptor;
    return;
  }
  uint8_t* out = work + d[kWorkOff];
  const long long n_out = g.filtered();
  Inflater s;
  s.init(streams + d[kStreamOff], d[kStreamLen], out, n_out, window);
  int st;
  for (;;) {
    long long at = 0;
    int len = 0, dist = 1;
    if (lane == 0) {
      st = s.run(tables, kWarpCopy);
      at = s.copy_at, len = s.copy_len, dist = s.copy_dist;
    }
    st = __shfl_sync(kFull, st, 0);
    if (st != kCopyPending) break;
    at = __shfl_sync(kFull, at, 0);
    len = __shfl_sync(kFull, len, 0);
    dist = __shfl_sync(kFull, dist, 0);
    __syncwarp();
    for (int j = lane; j < len; j += 32) s.put(at + j, s.source(at, dist, j));
    __syncwarp();
  }
  if (st == kOk) {
    // Adler-32 from per-lane chunks: s1 = 1 + sum s_k, s2 = n + sum (n - k) s_k; a chunk [lo, hi) contributes
    // sum (hi - k) s_k + (n - hi) sum s_k to the second.
    __syncwarp();
    const long long chunk = (n_out + 31) / 32, lo = min(n_out, lane * chunk), hi = min(n_out, lo + chunk);
    unsigned long long sum = 0, weighted = 0;
    for (long long k = lo; k < hi; ++k) {
      const uint32_t v = out[k];
      sum += v;
      weighted += (unsigned long long)(hi - k) * v;
    }
    unsigned long long s1 = sum % kAdlerMod;
    unsigned long long s2 = (weighted % kAdlerMod + (unsigned long long)((n_out - hi) % kAdlerMod) * s1) % kAdlerMod;
    for (int m = 16; m; m >>= 1) {
      s1 += __shfl_xor_sync(kFull, s1, m);
      s2 += __shfl_xor_sync(kFull, s2, m);
    }
    const uint32_t a = (uint32_t)((1 + s1) % kAdlerMod), b = (uint32_t)((n_out % kAdlerMod + s2) % kAdlerMod);
    const uint32_t trailer = __shfl_sync(kFull, s.adler, 0);
    if ((b << 16 | a) != trailer) st = kBadAdler;
  }
  if (lane == 0) status[f] = st;
}

__device__ __forceinline__ uint32_t paeth(uint32_t a, uint32_t b, uint32_t c) {
  const int p = (int)a + (int)b - (int)c;
  const int pa = abs(p - (int)a), pb = abs(p - (int)b), pc = abs(p - (int)c);
  return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}

__global__ void __launch_bounds__(kUnfilterThreads) unfilter_kernel(const int64_t* __restrict__ desc,
                                                                     uint8_t* __restrict__ work,
                                                                     uint8_t* __restrict__ images,
                                                                     int* __restrict__ status) {
  __shared__ int bad_filter;
  const int f = blockIdx.x, tid = threadIdx.x;
  if (status[f] != kOk) return;  // the whole block leaves
  const int64_t* d = desc + (size_t)f * kDescFields;
  Shape g;
  shape_of(d[kH], d[kW], d[kColourType], d[kBits], &g);  // checked by inflate_kernel
  uint8_t* s = work + d[kWorkOff];
  uint8_t* img = images + d[kOutOff];
  const long long seg = g.rowbytes + 1, steps_per_row = (g.rowbytes + g.bpp - 1) / g.bpp;
  const int bpp = g.bpp;
  const bool grey = d[kColourType] == 0;
  const int ppb = 8 / g.bits;  // pixels per byte of a sub-byte row
  const uint32_t mask = (1u << g.bits) - 1, scale = !grey || g.bits == 8 ? 1 : g.bits == 2 ? 85 : 17;
  if (tid == 0) bad_filter = 0;
  __syncthreads();
  for (long long band = 0; band < g.h; band += blockDim.x) {
    const long long y = band + tid;
    const long long rows = min((long long)blockDim.x, g.h - band);
    const bool active = y < g.h;
    uint8_t* row = s + y * seg + 1;
    const uint8_t* up = s + (y - 1) * seg + 1;
    int type = 0;
    if (active) {
      type = row[-1];
      if (type > 4) bad_filter = 1, type = 0;
    }
    const bool has_up = y > 0;
    const long long steps = steps_per_row + rows - 1;
    for (long long step = 0; step < steps; ++step) {
      const long long i = step - tid;
      if (active && i >= 0 && i < steps_per_row) {
        for (int q = 0; q < bpp; ++q) {
          const long long x = i * bpp + q;
          if (x >= g.rowbytes) break;
          const uint32_t a = x >= bpp ? row[x - bpp] : 0u;
          const uint32_t b = has_up ? up[x] : 0u;
          const uint32_t c = x >= bpp && has_up ? up[x - bpp] : 0u;
          uint32_t v = row[x];
          switch (type) {
            case 1: v += a; break;
            case 2: v += b; break;
            case 3: v += (a + b) >> 1; break;
            case 4: v += paeth(a, b, c); break;
            default: break;
          }
          v &= 0xffu;
          row[x] = (uint8_t)v;
          if (g.bits == 8) {
            img[y * g.rowbytes + x] = (uint8_t)v;
          } else {
            for (int t = 0; t < ppb; ++t) {
              const long long px = x * ppb + t;
              if (px < g.w) img[y * g.w + px] = (uint8_t)(((v >> (8 - g.bits * (t + 1))) & mask) * scale);
            }
          }
        }
      }
      __syncthreads();
    }
  }
  if (tid == 0 && bad_filter) status[f] = kBadFilter;
}

}  // namespace png_decode
}  // namespace b200

using namespace b200;

extern "C" {

DEVA_B200_API size_t deva_b200_png_decode_workspace_bytes(int h, int w, int colour_type, int bits) {
  png_decode::Shape g;
  if (!png_decode::shape_of(h, w, colour_type, bits, &g)) return 0;
  Carver<16> c{nullptr};
  c.take<uint8_t>(g.filtered());
  return c.bytes;
}

DEVA_B200_API int deva_b200_png_decode(const uint8_t* streams, const int64_t* desc, int n, uint8_t* out,
                                       void* workspace, int32_t* status, deva_stream_t stream) {
  B200_REQUIRE(n >= 0 && (n == 0 || (streams && desc && out && workspace && status)), "png_decode: bad arguments");
  if (n == 0) return 0;
  cudaStream_t s = S(stream);
  uint8_t* work = static_cast<uint8_t*>(workspace);
  B200_CUDA(cudaFuncSetAttribute(png_decode::inflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)png_decode::kInflateSmem));
  png_decode::inflate_kernel<<<n, 32, png_decode::kInflateSmem, s>>>(streams, desc, n, work, status);
  B200_LAUNCH_CHECK();
  png_decode::unfilter_kernel<<<n, png_decode::kUnfilterThreads, 0, s>>>(desc, work, out, status);
  B200_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
