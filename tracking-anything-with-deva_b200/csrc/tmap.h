// Host-side TMA tensor-map construction.  cuTensorMapEncodeTiled is a driver-API symbol;
// it is resolved at run time through the CUDA runtime so the library links (and loads on a
// GPU-less build box) without libcuda.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

enum class TmapType { F16, F32, BF16, U8 };

// Returns 0 on success; on failure returns non-zero and `err` points at a static message.
int make_tmap_2d(CUtensorMap* out, TmapType type, const void* base, uint64_t inner, uint64_t outer,
                 uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, const char** err);

// fp16 activation map for implicit-GEMM convolution: rank-5 dims (C, W, H, B, 1) with explicit element
// strides for W / H / B (so strided "phase" views of an NHWC buffer can be described), 128-byte swizzle,
// box (64, box_w, box_h, 1, 1).  Out-of-range coordinates (conv padding) are zero-filled.
int make_tmap_act5(CUtensorMap* out, const void* base, uint64_t c, uint64_t w, uint64_t h, uint64_t b,
                   long long stride_w, long long stride_h, long long stride_b, uint32_t box_w, uint32_t box_h,
                   const char** err);

// Same for an 8-bit (e4m3) tensor: dims (C bytes, W, H, B, 1), box (box_c, box_w, box_h, 1, 1), strides in bytes.
// box_c 128: 128-byte swizzle (the wgmma operand layout); box_c 64: unswizzled 64-byte rows.
int make_tmap_act5_u8(CUtensorMap* out, const void* base, uint64_t c, uint64_t w, uint64_t h, uint64_t b,
                      long long stride_w, long long stride_h, long long stride_b, uint32_t box_c, uint32_t box_w,
                      uint32_t box_h, const char** err);

// General rank-5 fp16 tiled map, 128-byte swizzle: dims / box in elements, strides (dims 1..4) in elements.
int make_tmap_f16_5d(CUtensorMap* out, const void* base, const uint64_t (&dims)[5], const long long (&strides)[4],
                     const uint32_t (&box)[5], const char** err);

// Im2col map of an NHWC tensor for stride-1 convolutions with `pad` pixels of zero padding: rank-4 dims (C, W, H, B),
// 128 pixels of box_c channels (box_c * element size = 128 B, 128-byte swizzle) per load.  A load at coordinates
// (c0, x - pad, y - pad, b) with im2col offsets (dx, dy) in [0, 2 pad] fetches, for the 128 consecutive output pixels
// that start at (y, x) of image b in row-major order, input pixel (y' - pad + dy, x' - pad + dx) of each; rows past
// the image continue into the next one, and everything outside the tensor is zero-filled.
int make_tmap_im2col4(CUtensorMap* out, TmapType type, const void* base, uint64_t c, uint64_t w, uint64_t h, uint64_t b,
                      uint32_t box_c, int pad, const char** err);

}  // namespace b200
