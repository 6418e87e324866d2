#include "tmap.h"

#include <mutex>

namespace b200 {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

// The driver entry point `Name`, resolved once through the runtime (no libcuda link).
template <typename Fn>
static Fn resolve_driver(const char* name, const char* missing, const char** err) {
  static Fn fn = nullptr;
  static std::once_flag once;
  static const char* failure = nullptr;
  std::call_once(once, [&] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) {
      failure = missing;
      (void)cudaGetLastError();
    } else {
      fn = reinterpret_cast<Fn>(p);
    }
  });
  if (!fn && err) *err = failure;
  return fn;
}
static EncodeTiledFn resolve_encode(const char** err) {
  return resolve_driver<EncodeTiledFn>("cuTensorMapEncodeTiled", "cuTensorMapEncodeTiled not available (no CUDA driver?)",
                                       err);
}
static EncodeIm2colFn resolve_encode_im2col(const char** err) {
  return resolve_driver<EncodeIm2colFn>("cuTensorMapEncodeIm2col",
                                        "cuTensorMapEncodeIm2col not available (no CUDA driver?)", err);
}

static CUtensorMapDataType to_cu(TmapType t, uint32_t* esize) {
  switch (t) {
    case TmapType::F16: *esize = 2; return CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    case TmapType::BF16: *esize = 2; return CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    case TmapType::U8: *esize = 1; return CU_TENSOR_MAP_DATA_TYPE_UINT8;
    default: *esize = 4; return CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  }
}

int make_tmap_2d(CUtensorMap* out, TmapType type, const void* base, uint64_t inner, uint64_t outer,
                 uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, const char** err) {
  EncodeTiledFn fn = resolve_encode(err);
  if (!fn) return 1;
  uint32_t esize;
  CUtensorMapDataType dt = to_cu(type, &esize);
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (row_stride_bytes & 15) || box_inner * esize != 128 ||
      box_outer > 256 || inner == 0 || outer == 0) {
    if (err) *err = "make_tmap_2d: bad alignment / box";
    return 2;
  }
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstride[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, dt, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    if (err) *err = "cuTensorMapEncodeTiled(2d) failed";
    return 3;
  }
  return 0;
}

int make_tmap_f16_5d(CUtensorMap* out, const void* base, const uint64_t (&dims)[5], const long long (&strides)[4],
                     const uint32_t (&box)[5], const char** err) {
  EncodeTiledFn fn = resolve_encode(err);
  if (!fn) return 1;
  bool bad = (reinterpret_cast<uintptr_t>(base) & 15) != 0 || box[0] * 2 > 128;
  cuuint64_t gdim[5], gstride[4];
  cuuint32_t bx[5], estr[5] = {1, 1, 1, 1, 1};
  for (int i = 0; i < 5; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; bad |= dims[i] == 0 || box[i] == 0 || box[i] > 256; }
  for (int i = 0; i < 4; ++i) { gstride[i] = (cuuint64_t)strides[i] * 2; bad |= (strides[i] & 7) != 0 || strides[i] <= 0; }
  if (bad) {
    if (err) *err = "make_tmap_f16_5d: bad alignment / box";
    return 2;
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(base), gdim, gstride, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    if (err) *err = "cuTensorMapEncodeTiled(5d) failed";
    return 3;
  }
  return 0;
}

int make_tmap_act5_u8(CUtensorMap* out, const void* base, uint64_t c, uint64_t w, uint64_t h, uint64_t b,
                      long long stride_w, long long stride_h, long long stride_b, uint32_t box_c, uint32_t box_w,
                      uint32_t box_h, const char** err) {
  EncodeTiledFn fn = resolve_encode(err);
  if (!fn) return 1;
  const long long strides[4] = {stride_w, stride_h, stride_b, stride_b * (long long)b};
  bool bad = (reinterpret_cast<uintptr_t>(base) & 15) != 0 || (box_c != 128 && box_c != 64) || c < box_c || box_w == 0 ||
             box_h == 0 || box_w > 256 || box_h > 256;
  cuuint64_t gdim[5] = {c, w, h, b, 1}, gstride[4];
  cuuint32_t bx[5] = {box_c, box_w, box_h, 1, 1}, estr[5] = {1, 1, 1, 1, 1};
  for (int i = 0; i < 4; ++i) { gstride[i] = (cuuint64_t)strides[i]; bad |= (strides[i] & 15) != 0 || strides[i] <= 0; }
  if (bad) {
    if (err) *err = "make_tmap_act5_u8: bad alignment / box";
    return 2;
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 5, const_cast<void*>(base), gdim, gstride, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, box_c == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    if (err) *err = "cuTensorMapEncodeTiled(5d u8) failed";
    return 3;
  }
  return 0;
}

int make_tmap_act5(CUtensorMap* out, const void* base, uint64_t c, uint64_t w, uint64_t h, uint64_t b,
                   long long stride_w, long long stride_h, long long stride_b, uint32_t box_w, uint32_t box_h,
                   const char** err) {
  if (c < 64) {
    if (err) *err = "make_tmap_act5: needs >= 64 channels";
    return 2;
  }
  const uint64_t dims[5] = {c, w, h, b, 1};
  const long long strides[4] = {stride_w, stride_h, stride_b, stride_b * (long long)b};
  const uint32_t box[5] = {64, box_w, box_h, 1, 1};
  return make_tmap_f16_5d(out, base, dims, strides, box, err);
}

int make_tmap_im2col4(CUtensorMap* out, TmapType type, const void* base, uint64_t c, uint64_t w, uint64_t h, uint64_t b,
                      uint32_t box_c, int pad, const char** err) {
  EncodeIm2colFn fn = resolve_encode_im2col(err);
  if (!fn) return 1;
  uint32_t esize;
  const CUtensorMapDataType dt = to_cu(type, &esize);
  const uint64_t row = c * esize;
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (row & 15) || box_c * esize != 128 || c < box_c || w == 0 || h == 0 ||
      b == 0 || pad < 0 || pad > 127) {
    if (err) *err = "make_tmap_im2col4: bad alignment / box";
    return 2;
  }
  cuuint64_t gdim[4] = {c, w, h, b};
  cuuint64_t gstride[3] = {row, row * w, row * w * h};
  // base pixels (the filter window's top-left input pixel) span [-pad, dim - 1 - pad] in W and H
  const int lower[2] = {-pad, -pad}, upper[2] = {-pad, -pad};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(out, dt, 4, const_cast<void*>(base), gdim, gstride, lower, upper, box_c, 128, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    if (err) *err = "cuTensorMapEncodeIm2col failed";
    return 3;
  }
  return 0;
}

}  // namespace b200
