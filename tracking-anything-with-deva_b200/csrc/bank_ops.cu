// Memory-bank data movement: operand packing, O(1) append, compaction gathers.
// Reference behaviour replaced: KeyValueMemoryStore.add / sieve_by_range / remove_obsolete_features
// (deva/inference/kv_memory_store.py:35-185), which re-allocates and copies the whole bank with torch.cat
// on every memory frame.  Here the bank is preallocated token-major and these kernels touch only the
// tokens that change.  All kernels are HBM-bound copy/convert passes.
#include <cuda_fp16.h>

#include "common.h"

namespace b200 {
namespace bank {

constexpr int TOK = 32;  // tokens per block

__device__ __forceinline__ void split_store(float x, __half* hi, __half* lo, long long off) {
  const __half h = __float2half_rn(x);
  hi[off] = h;
  lo[off] = __float2half_rn(x - __half2float(h));
}

// Packs query rows  [ -qe | 2*qk*qe ]  as fp16 (hi, lo) and bsq[q] = sum_c qe*qk^2
// (operands of memory_utils.py:30-32).  Input element (c, q) lives at c*sc + q*sq.
template <int CK>
__global__ void __launch_bounds__(256)
pack_query_kernel(const float* __restrict__ qk, const float* __restrict__ qe, long long sc, long long sq, int q,
                  __half* __restrict__ hi, __half* __restrict__ lo, float* __restrict__ bsq) {
  __shared__ float sk[TOK][CK + 1], se[TOK][CK + 1];
  const int q0 = blockIdx.x * TOK;
  for (int i = threadIdx.x; i < TOK * CK; i += 256) {
    int t, c;
    if (sq == 1) { t = i % TOK; c = i / TOK; } else { c = i % CK; t = i / CK; }
    const int qi = q0 + t;
    float k = 0.f, e = 0.f;
    if (qi < q) { k = qk[c * sc + qi * sq]; e = qe[c * sc + qi * sq]; }
    sk[t][c] = k;
    se[t][c] = e;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < TOK * 2 * CK; i += 256) {
    const int t = i / (2 * CK), col = i % (2 * CK);
    if (q0 + t >= q) continue;
    const float v = (col < CK) ? -se[t][col] : 2.f * sk[t][col - CK] * se[t][col - CK];
    split_store(v, hi, lo, (long long)(q0 + t) * (2 * CK) + col);
  }
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t = w; t < TOK; t += 8) {
    float a = 0.f;
    for (int c = lane; c < CK; c += 32) a += se[t][c] * sk[t][c] * sk[t][c];
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0 && q0 + t < q) bsq[q0 + t] = a;
  }
}

// Packs memory-key rows  [ s*mk^2 | s*mk ]  (s = shrinkage / sqrt(CK)) as fp16 (hi, lo), neg_s = -s,
// and token-major fp32 copies of key / selection / shrinkage.  kv_memory_store.py:97-116.
template <int CK>
__global__ void __launch_bounds__(256)
pack_keys_kernel(const float* __restrict__ key, const float* __restrict__ sel, long long sc, long long sn,
                 const float* __restrict__ shr, int n, __half* __restrict__ hi, __half* __restrict__ lo,
                 float* __restrict__ neg_s, float* __restrict__ raw_key, float* __restrict__ raw_sel,
                 float* __restrict__ raw_shr) {
  __shared__ float sk[TOK][CK + 1], se[TOK][CK + 1];
  __shared__ float ss[TOK];
  const int n0 = blockIdx.x * TOK;
  const float inv = rsqrtf((float)CK);
  for (int i = threadIdx.x; i < TOK * CK; i += 256) {
    int t, c;
    if (sn == 1) { t = i % TOK; c = i / TOK; } else { c = i % CK; t = i / CK; }
    const int ni = n0 + t;
    sk[t][c] = (ni < n) ? key[c * sc + ni * sn] : 0.f;
    if (sel) se[t][c] = (ni < n) ? sel[c * sc + ni * sn] : 0.f;
  }
  if (threadIdx.x < TOK) ss[threadIdx.x] = (n0 + threadIdx.x < n) ? shr[n0 + threadIdx.x] : 0.f;
  __syncthreads();
  for (int i = threadIdx.x; i < TOK * 2 * CK; i += 256) {
    const int t = i / (2 * CK), col = i % (2 * CK);
    if (n0 + t >= n) continue;
    const float s = ss[t] * inv;
    const float k = sk[t][col < CK ? col : col - CK];
    split_store((col < CK) ? s * k * k : s * k, hi, lo, (long long)(n0 + t) * (2 * CK) + col);
    if (col < CK) {
      raw_key[(long long)(n0 + t) * CK + col] = k;
      if (sel) raw_sel[(long long)(n0 + t) * CK + col] = se[t][col];
    }
  }
  if (threadIdx.x < TOK && n0 + threadIdx.x < n) {
    neg_s[n0 + threadIdx.x] = -ss[threadIdx.x] * inv;
    raw_shr[n0 + threadIdx.x] = ss[threadIdx.x];
  }
}

// fp32 [rows, n] (ld_src) -> fp16 bank block dst[row, col0 + j] (ld_dst).  memory_manager.py:199-205.
__global__ void __launch_bounds__(256)
append_values_kernel(const float* __restrict__ src, long long ld_src, __half* __restrict__ dst, long long ld_dst,
                     int rows, int n) {
  const long long total = (long long)rows * n;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long r = i / n;
    const int j = (int)(i - r * n);
    dst[r * ld_dst + j] = __float2half_rn(src[r * ld_src + j]);
  }
}

// dst row i = src row idx[i]; rows are row_bytes long (multiple of 16).
__global__ void __launch_bounds__(256)
gather_rows_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src, const int* __restrict__ idx, int n,
                   int vec_per_row) {
  const long long total = (long long)n * vec_per_row;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long r = i / vec_per_row;
    const int v = (int)(i - r * vec_per_row);
    dst[i] = src[(long long)idx[r] * vec_per_row + v];
  }
}
__global__ void __launch_bounds__(256)
gather_f32_kernel(float* __restrict__ dst, const float* __restrict__ src, const int* __restrict__ idx, int n) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}
// dst[r, i] = src[r, idx[i]]  (value bank columns)
__global__ void __launch_bounds__(256)
gather_cols_f16_kernel(__half* __restrict__ dst, long long ld_dst, const __half* __restrict__ src, long long ld_src,
                       const int* __restrict__ idx, int rows, int n) {
  const long long total = (long long)rows * n;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long r = i / n;
    const int j = (int)(i - r * n);
    dst[r * ld_dst + j] = src[r * ld_src + idx[j]];
  }
}
// usage[i] = use[i] / life[i]  (kv_memory_store.py:187-193)
__global__ void __launch_bounds__(256)
usage_kernel(float* __restrict__ out, const float* __restrict__ use, const float* __restrict__ life, int n) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < n) out[i] = use[i] / life[i];
}

}  // namespace bank

static int grid_for(long long total) {
  long long g = (total + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace b200

using namespace b200;

extern "C" {

DEVA_B200_API int deva_b200_pack_query(const float* qk, const float* qe, int64_t stride_c, int64_t stride_q, int ck, int q,
                                       void* q_hi, void* q_lo, float* bsq, deva_stream_t stream) {
  B200_REQUIRE(q >= 1, "pack_query: empty");
  __half* hi = H(q_hi);
  __half* lo = H(q_lo);
  const cudaStream_t s = S(stream);
  const int grid = ceil_div(q, bank::TOK);
  if (ck == 64) bank::pack_query_kernel<64><<<grid, 256, 0, s>>>(qk, qe, stride_c, stride_q, q, hi, lo, bsq);
  else if (ck == 32) bank::pack_query_kernel<32><<<grid, 256, 0, s>>>(qk, qe, stride_c, stride_q, q, hi, lo, bsq);
  else B200_REQUIRE(false, "pack_query: key_dim %d unsupported (32 or 64)", ck);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_pack_keys(const float* key, const float* selection, int64_t stride_c, int64_t stride_t,
                                      const float* shrinkage, int ck, int n, void* k_hi, void* k_lo, float* neg_s,
                                      float* raw_key, float* raw_sel, float* raw_shr, deva_stream_t stream) {
  B200_REQUIRE(n >= 1, "pack_keys: empty");
  B200_REQUIRE(selection == nullptr || raw_sel != nullptr, "pack_keys: selection given without a destination");
  __half* hi = H(k_hi);
  __half* lo = H(k_lo);
  const cudaStream_t s = S(stream);
  const int grid = ceil_div(n, bank::TOK);
  if (ck == 64)
    bank::pack_keys_kernel<64><<<grid, 256, 0, s>>>(key, selection, stride_c, stride_t, shrinkage, n, hi, lo, neg_s,
                                                    raw_key, raw_sel, raw_shr);
  else if (ck == 32)
    bank::pack_keys_kernel<32><<<grid, 256, 0, s>>>(key, selection, stride_c, stride_t, shrinkage, n, hi, lo, neg_s,
                                                    raw_key, raw_sel, raw_shr);
  else B200_REQUIRE(false, "pack_keys: key_dim %d unsupported (32 or 64)", ck);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_append_values(const float* src, int64_t ld_src, void* dst, int64_t ld_dst, int rows, int n,
                                          deva_stream_t stream) {
  B200_REQUIRE(rows >= 1 && n >= 1, "append_values: empty");
  bank::append_values_kernel<<<grid_for((long long)rows * n), 256, 0, S(stream)>>>(src, ld_src, H(dst), ld_dst, rows, n);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_gather_rows(void* dst, const void* src, const int32_t* idx, int n, int row_bytes,
                                        deva_stream_t stream) {
  B200_REQUIRE(row_bytes % 16 == 0, "gather_rows: row_bytes %d not a multiple of 16", row_bytes);
  if (n <= 0) return 0;
  const int vec = row_bytes / 16;
  bank::gather_rows_kernel<<<grid_for((long long)n * vec), 256, 0, S(stream)>>>(
      reinterpret_cast<uint4*>(dst), reinterpret_cast<const uint4*>(src), idx, n, vec);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_gather_f32(float* dst, const float* src, const int32_t* idx, int n, deva_stream_t stream) {
  if (n <= 0) return 0;
  bank::gather_f32_kernel<<<ceil_div(n, 256), 256, 0, S(stream)>>>(dst, src, idx, n);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_gather_cols_f16(void* dst, int64_t ld_dst, const void* src, int64_t ld_src, const int32_t* idx,
                                            int rows, int n, deva_stream_t stream) {
  if (n <= 0 || rows <= 0) return 0;
  bank::gather_cols_f16_kernel<<<grid_for((long long)rows * n), 256, 0, S(stream)>>>(H(dst), ld_dst, H(src), ld_src, idx,
                                                                                     rows, n);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_usage(float* out, const float* use_cnt, const float* life_cnt, int n, deva_stream_t stream) {
  if (n <= 0) return 0;
  bank::usage_kernel<<<ceil_div(n, 256), 256, 0, S(stream)>>>(out, use_cnt, life_cnt, n);
  B200_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
