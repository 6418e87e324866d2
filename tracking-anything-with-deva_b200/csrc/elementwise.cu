// HBM-bound helper kernels of the NHWC fp16 network path: layout/precision conversion at the API boundary,
// max-pool, bilinear x2 + skip add, area down-sampling, CBAM (reference deva/model/cbam.py:21-77), and the
// soft-aggregation / x4 upsampling / softmax tail (network.py:33-40,144-168).  One thread per output element (or per
// pixel x channel-vector); all accesses are coalesced along the channel axis.
#include <algorithm>
#include <climits>
#include <cuda_fp16.h>
#include <math_constants.h>
#include <stdint.h>

#include "common.h"

namespace b200 {
namespace ew {

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ void ld8(const __half* p, float (&f)[8]) {
  const uint4 v = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int e = 0; e < 4; ++e) { const float2 t = __half22float2(h[e]); f[2 * e] = t.x; f[2 * e + 1] = t.y; }
}
__device__ __forceinline__ void st8(__half* p, const float (&f)[8], bool relu) {
  uint4 v;
  __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
  for (int e = 0; e < 4; ++e)
    h[e] = relu ? __floats2half2_rn(fmaxf(f[2 * e], 0.f), fmaxf(f[2 * e + 1], 0.f)) : __floats2half2_rn(f[2 * e], f[2 * e + 1]);
  *reinterpret_cast<uint4*>(p) = v;
}

// ---------------------------------------------------------------- layout conversion
// fp32 NCHW [B,C,H,W] -> fp16 NHWC [B,H,W,Cp] (channels >= C are zero)
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, __half* __restrict__ dst, int B, int C, int H, int W,
                                    int Cp) {
  const long long total = (long long)B * H * W * Cp;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % Cp);
    long long p = i / Cp;
    const int x = (int)(p % W); p /= W;
    const int y = (int)(p % H);
    const int b = (int)(p / H);
    dst[i] = (c < C) ? __float2half_rn(src[(((long long)b * C + c) * H + y) * W + x]) : __float2half_rn(0.f);
  }
}
// im2col for the 7x7 stride-2 pad-3 stems (resnet.py:120): planes fp32 [B, C, H, W] -> fp16 [B, H/2, W/2, Kp]
// with column k = (kh*7 + kw)*C + c for k < 49*C and zeros up to Kp (a multiple of 64).  The stem then runs
// as a 1x1 implicit GEMM over Kp "channels" on the tensor cores.
constexpr int IM_XT = 64;  // output columns per block
__global__ void __launch_bounds__(256)
stem_im2col_kernel(const float* __restrict__ src, __half* __restrict__ dst, __half* __restrict__ dst_lo,
                   int B, int C, int H, int W, int Kp) {
  // Block = (image b, output row yo, IM_XT output columns).  The 7 input rows x (2*IM_XT + 5) input columns of all C
  // planes are staged in shared memory with coalesced loads; each thread then emits 8 consecutive im2col columns
  // (one 16-byte store for the fp16 values, one for the remainders).
  extern __shared__ float patch[];  // [C][7][PW]
  const int Ho = H / 2, Wo = W / 2;
  constexpr int PW = 2 * IM_XT + 5;
  const int b = blockIdx.y / Ho, yo = blockIdx.y - b * Ho;
  const int xo0 = blockIdx.x * IM_XT;
  const int x_in0 = 2 * xo0 - 3, y_in0 = 2 * yo - 3;
  const float* img = src + (long long)b * C * H * W;
  for (int i = threadIdx.x; i < C * 7 * PW; i += 256) {
    const int px = i % PW, r = (i / PW) % 7, c = i / (7 * PW);
    const int y = y_in0 + r, x = x_in0 + px;
    patch[i] = (y >= 0 && y < H && x >= 0 && x < W) ? img[((long long)c * H + y) * W + x] : 0.f;
  }
  __syncthreads();
  const int nx = min(IM_XT, Wo - xo0);
  const long long out_base = (((long long)b * Ho + yo) * Wo + xo0) * Kp;
  const int kreal = 49 * C, K8 = Kp / 8;
  for (int i = threadIdx.x; i < nx * K8; i += 256) {
    const int xl = i / K8, k0 = (i - xl * K8) * 8;
    float v[8], r[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = k0 + e;
      float x = 0.f;
      if (k < kreal) {
        const int tap = k / C, c = k - tap * C;
        const int ky = tap / 7, kx = tap - ky * 7;
        x = patch[(c * 7 + ky) * PW + 2 * xl + kx];
      }
      v[e] = x;
      r[e] = x - __half2float(__float2half_rn(x));
    }
    st8(dst + out_base + (long long)xl * Kp + k0, v, false);
    if (dst_lo) st8(dst_lo + out_base + (long long)xl * Kp + k0, r, false);
  }
}

// Block variant for the shapes the network uses (C = 1: mask planes, Kp = 64; C = 3: image, Kp = 192, with or without
// the fp16 remainders).  The generic kernel spends ~120 instructions of index arithmetic per 16-byte store and ran at
// 16-28 % of the HBM peak.  Here a block stages the patch under IM1_XT output pixels x ROWS output rows in shared memory
// (even / odd input columns de-interleaved), with a table of each column's patch offset.  The block's output in one row
// is nx * Kp contiguous halves, and thread t writes its 16-byte pieces t, t + IM1_XT, ...: a warp stores 512
// contiguous bytes per instruction.  (With one pixel per thread, a warp's 16-byte stores were 32 pieces Kp * 2 bytes
// apart, and the kernel wrote the pixel encoder's 400 MB of columns at about a fifth of the HBM bandwidth.)  Same values
// as the generic kernel.
constexpr int IM1_XT = 128;
template <int C, int ROWS, bool LO>
__global__ void __launch_bounds__(IM1_XT)
stem_im2col_px_kernel(const float* __restrict__ src, __half* __restrict__ dst, __half* __restrict__ dst_lo, int B, int H, int W) {
  constexpr int PR = 2 * ROWS + 5;      // input rows under ROWS output rows
  constexpr int PH = IM1_XT + 3;        // input column x_in0 + 2*i (+1) for i in [0, PH)
  constexpr int KP = (49 * C + 63) / 64 * 64;
  constexpr int K8 = KP / 8;            // 16-byte pieces of one pixel's row
  __shared__ float patch[2][C][PR][PH];  // [input column parity][plane][row][column / 2]
  __shared__ __align__(16) int tab[KP];  // column k = (ky*7 + kx)*C + c -> its offset in patch for output (row 0, pixel 0)
  const int Ho = H / 2, Wo = W / 2;
  const int groups = (Ho + ROWS - 1) / ROWS;
  const int b = blockIdx.y / groups, yo0 = (blockIdx.y - b * groups) * ROWS;
  const int xo0 = blockIdx.x * IM1_XT;
  const int x_in0 = 2 * xo0 - 3, y_in0 = 2 * yo0 - 3;
  const float* img = src + (long long)b * C * H * W;
  for (int i = threadIdx.x; i < C * PR * 2 * PH; i += IM1_XT) {
    const int px = i % (2 * PH), r = (i / (2 * PH)) % PR, c = i / (2 * PH * PR);
    const int y = y_in0 + r, x = x_in0 + px;
    patch[px & 1][c][r][px >> 1] = (y >= 0 && y < H && x >= 0 && x < W) ? img[((long long)c * H + y) * W + x] : 0.f;
  }
  for (int k = threadIdx.x; k < KP; k += IM1_XT) {
    const int tap = k / C, c = k - tap * C, ky = tap / 7, kx = tap - ky * 7;
    tab[k] = k < 49 * C ? &patch[kx & 1][c][ky][kx >> 1] - &patch[0][0][0][0] : -1;
  }
  __syncthreads();
  const float* pf = &patch[0][0][0][0];
  const int nx = min(IM1_XT, Wo - xo0);
#pragma unroll 1
  for (int rr = 0; rr < ROWS; ++rr) {
    const int yo = yo0 + rr;
    if (yo >= Ho) break;
    const long long out = (((long long)b * Ho + yo) * Wo + xo0) * KP;
#pragma unroll 2
    for (int j = threadIdx.x; j < nx * K8; j += IM1_XT) {  // piece j: pixel xo0 + j / K8, columns 8 (j % K8) + 0..7
      const int xl = j / K8, k0 = (j - xl * K8) * 8;
      const int base = 2 * rr * PH + xl;
      const int4 t0 = *reinterpret_cast<const int4*>(tab + k0), t1 = *reinterpret_cast<const int4*>(tab + k0 + 4);
      const int t[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
      uint4 oh, ol;
      __half2* h2 = reinterpret_cast<__half2*>(&oh);
      __half2* l2 = reinterpret_cast<__half2*>(&ol);
#pragma unroll
      for (int k2 = 0; k2 < 4; ++k2) {
        const float v0 = t[2 * k2] >= 0 ? pf[t[2 * k2] + base] : 0.f;
        const float v1 = t[2 * k2 + 1] >= 0 ? pf[t[2 * k2 + 1] + base] : 0.f;
        h2[k2] = __floats2half2_rn(v0, v1);
        if (LO) {
          const float2 back = __half22float2(h2[k2]);
          l2[k2] = __floats2half2_rn(v0 - back.x, v1 - back.y);
        }
      }
      reinterpret_cast<uint4*>(dst + out)[j] = oh;
      if (LO) reinterpret_cast<uint4*>(dst_lo + out)[j] = ol;
    }
  }
}

// ---------------------------------------------------------------- pooling / resampling (NHWC fp16, 8 channels per thread)
// 3x3 stride-2 pad-1 max pool (resnet.py:123)
__global__ void maxpool_kernel(const __half* __restrict__ x, const __half* __restrict__ x_lo, __half* __restrict__ y,
                               __half* __restrict__ y_lo, int B, int H, int W, int C) {
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2, C8 = C / 8;
  const long long total = (long long)B * Ho * Wo * C8;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % C8) * 8;
    long long p = i / C8;
    const int xo = (int)(p % Wo); p /= Wo;
    const int yo = (int)(p % Ho);
    const int b = (int)(p / Ho);
    float m[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) m[e] = -CUDART_INF_F;
    for (int dy = -1; dy <= 1; ++dy) {
      const int yy = 2 * yo + dy;
      if (yy < 0 || yy >= H) continue;
      for (int dx = -1; dx <= 1; ++dx) {
        const int xx = 2 * xo + dx;
        if (xx < 0 || xx >= W) continue;
        float f[8];
        const long long o = (((long long)b * H + yy) * W + xx) * C + c;
        ld8(x + o, f);
        if (x_lo) {
          float l[8];
          ld8(x_lo + o, l);
#pragma unroll
          for (int e = 0; e < 8; ++e) f[e] += l[e];
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) m[e] = fmaxf(m[e], f[e]);
      }
    }
    const long long oo = (((long long)b * Ho + yo) * Wo + xo) * C + c;
    st8(y + oo, m, false);
    if (y_lo) {
      float r[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) r[e] = m[e] - __half2float(__float2half_rn(m[e]));
      st8(y_lo + oo, r, false);
    }
  }
}

// out = bilinear_x2(g) + skip (skip is one image broadcast over the batch; MaskUpsampleBlock: upsample_groups +
// distributor 'add', modules.py:88-91) on the residual stream carried as fp16 hi/lo pairs (DESIGN section 4 "precision
// plan"): g = g + g_lo and skip = skip + skip_lo on input; the raw sum is written as (hi, lo), the ReLU'd copy - an MMA
// operand only - as hi.
__device__ __forceinline__ void st8_split(__half* hi, __half* lo, const float (&f)[8]) {
  uint4 vh, vl;
  __half2* h2 = reinterpret_cast<__half2*>(&vh);
  __half2* l2 = reinterpret_cast<__half2*>(&vl);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    h2[e] = __floats2half2_rn(f[2 * e], f[2 * e + 1]);
    const float2 back = __half22float2(h2[e]);
    l2[e] = __floats2half2_rn(f[2 * e] - back.x, f[2 * e + 1] - back.y);
  }
  *reinterpret_cast<uint4*>(hi) = vh;
  *reinterpret_cast<uint4*>(lo) = vl;
}
__global__ void __launch_bounds__(256)
up2_add_split_kernel(const __half* __restrict__ g, const __half* __restrict__ g_lo, const __half* __restrict__ skip,
                     const __half* __restrict__ skip_lo, __half* __restrict__ raw, __half* __restrict__ raw_lo,
                     __half* __restrict__ relu, unsigned char* __restrict__ relu_lo8, int B, int h, int w, int C) {
  // A thread owns 8 channels of the 2 x 2 OUTPUT block {2k-1, 2k} x {2j-1, 2j}: with align_corners = False these four
  // pixels interpolate between the same four source pixels (rows k-1, k / columns j-1, j, clamped at the border) with
  // weights 0.25 / 0.75, so the source quad (hi + lo) is loaded once per four outputs and there is no serial walk:
  // every thread is one independent load -> compute -> store chain (the row-walking version kept the DRAM traffic at the
  // algorithmic 1x but ran at half the HBM rate: eight dependent rows per thread; the per-pixel version before it re-read
  // the source 5x).  blockIdx.y = (k, image), k in [0, h]; the clamped border blocks produce the reference's values
  // exactly (a + (a - a) * wx == a).  The image index runs fastest: the B blocks of one k read the same two skip rows
  // back to back, so the broadcast skip (hi + lo, 134 MB at 1/4 of 1080p with 256 channels) comes from DRAM about once
  // instead of once per image, and stays in L2 for the others.
  const int H = 2 * h, W = 2 * w, C8 = C / 8;
  const int k = blockIdx.y / B, b = blockIdx.y - k * B;
  const int ya = max(k - 1, 0), yb = min(k, h - 1);
  const int row_vecs = (w + 1) * C8;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < row_vecs; i += gridDim.x * 256) {
    const int j = i / C8, c = (i - j * C8) * 8;
    const int xa = max(j - 1, 0), xb = min(j, w - 1);
    float qa[8], qb[8], qc[8], qd[8], l[8];  // source quad: (ya, xa), (ya, xb), (yb, xa), (yb, xb)
    const long long oa = (((long long)b * h + ya) * w) * C + c, ob = (((long long)b * h + yb) * w) * C + c;
    auto load = [&](const long long o, float (&q)[8]) {
      ld8(g + o, q);
      ld8(g_lo + o, l);
#pragma unroll
      for (int e = 0; e < 8; ++e) q[e] += l[e];
    };
    load(oa + (long long)xa * C, qa);
    load(oa + (long long)xb * C, qb);
    load(ob + (long long)xa * C, qc);
    load(ob + (long long)xb * C, qd);
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const int Y = 2 * k - 1 + dy;
      if (Y < 0 || Y >= H) continue;
      const float wy = dy ? 0.75f : 0.25f;
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int X = 2 * j - 1 + dx;
        if (X < 0 || X >= W) continue;
        const float wx = dx ? 0.75f : 0.25f;
        float o[8], s_[8];
        ld8(skip + ((long long)Y * W + X) * C + c, s_);
        ld8(skip_lo + ((long long)Y * W + X) * C + c, l);
#pragma unroll
        for (int e = 0; e < 8; ++e) s_[e] += l[e];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float top = qa[e] + (qb[e] - qa[e]) * wx, bot = qc[e] + (qd[e] - qc[e]) * wx;
          o[e] = top + (bot - top) * wy + s_[e];
        }
        const long long off = (((long long)b * H + Y) * W + X) * C + c;
        st8_split(raw + off, raw_lo + off, o);
        if (relu_lo8) {  // low-order part as e4m3 of (x - fp16(x)) * 4096: operand of an fp8 correction pass
          uint32_t w8[2];
#pragma unroll
          for (int e = 0; e < 8; ++e) o[e] = fmaxf(o[e], 0.f);
          st8(relu + off, o, false);
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float q4[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) q4[t] = (o[4 * e + t] - __half2float(__float2half_rn(o[4 * e + t]))) * 4096.f;
            unsigned short a16, b16;
            asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(a16) : "f"(q4[1]), "f"(q4[0]));
            asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(b16) : "f"(q4[3]), "f"(q4[2]));
            w8[e] = (uint32_t)a16 | ((uint32_t)b16 << 16);
          }
          *reinterpret_cast<uint2*>(relu_lo8 + off) = make_uint2(w8[0], w8[1]);
        } else if (relu) {
          st8(relu + off, o, true);
        }
      }
    }
  }
}

// r x r average pooling (F.interpolate mode='area' with an integer ratio), NHWC fp16
__global__ void area_down_kernel(const __half* __restrict__ x, __half* __restrict__ y, int B, int H, int W, int C, int r) {
  const int Ho = H / r, Wo = W / r, C8 = C / 8;
  const long long total = (long long)B * Ho * Wo * C8;
  const float inv = 1.f / (r * r);
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % C8) * 8;
    long long p = i / C8;
    const int xo = (int)(p % Wo); p /= Wo;
    const int yo = (int)(p % Ho);
    const int b = (int)(p / Ho);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int dy = 0; dy < r; ++dy)
      for (int dx = 0; dx < r; ++dx) {
        float f[8];
        ld8(x + (((long long)b * H + yo * r + dy) * W + xo * r + dx) * C + c, f);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += f[e];
      }
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] *= inv;
    st8(y + (((long long)b * Ho + yo) * Wo + xo) * C + c, acc, false);
  }
}
// same for single-channel fp32 planes [B,H,W] -> [B,H/r,W/r]
__global__ void area_down_plane_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int r) {
  const int Ho = H / r, Wo = W / r;
  const long long total = (long long)B * Ho * Wo;
  const float inv = 1.f / (r * r);
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int xo = (int)(i % Wo);
    long long p = i / Wo;
    const int yo = (int)(p % Ho);
    const int b = (int)(p / Ho);
    float acc = 0.f;
    for (int dy = 0; dy < r; ++dy)
      for (int dx = 0; dx < r; ++dx) acc += x[((long long)b * H + yo * r + dy) * W + xo * r + dx];
    y[i] = acc * inv;
  }
}

// ---------------------------------------------------------------- CBAM (cbam.py:21-77)
// per (image, channel) partial sum and max over a slice of the pixels.  grid (B, kPoolSplit), 256 threads: a thread owns
// 8 channels (one 16-byte load per pixel and operand) and every (256 / (C/8))-th pixel of the slice; the pixel lanes are
// folded through shared memory.  (The one-channel-per-thread version issued 2-byte loads: 64 bytes per warp instruction.)
constexpr int kPoolSplit = 64;
__global__ void __launch_bounds__(256)
cbam_pool_kernel(const __half* __restrict__ x, const __half* __restrict__ x_lo, float* __restrict__ psum,
                 float* __restrict__ pmax, int HW, int C) {
  __shared__ float ss[256 * 8], sm[256 * 8];
  const int b = blockIdx.x, sp = blockIdx.y;
  const int C8 = C / 8, lanes = 256 / C8;  // pixel lanes (host guarantees 256 % C8 == 0)
  const int cv = threadIdx.x % C8, pl = threadIdx.x / C8;
  const int per = (HW + kPoolSplit - 1) / kPoolSplit;
  const int i0 = sp * per, i1 = min(HW, i0 + per);
  float s[8], m[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { s[e] = 0.f; m[e] = -CUDART_INF_F; }
  for (int i = i0 + pl; i < i1; i += lanes) {
    const long long o = ((long long)b * HW + i) * C + cv * 8;
    float v[8], l[8];
    ld8(x + o, v);
    ld8(x_lo + o, l);
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] += l[e];
#pragma unroll
    for (int e = 0; e < 8; ++e) { s[e] += v[e]; m[e] = fmaxf(m[e], v[e]); }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) { ss[e * 256 + threadIdx.x] = s[e]; sm[e * 256 + threadIdx.x] = m[e]; }
  __syncthreads();
  if (pl == 0) {
    for (int q = 1; q < lanes; ++q) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        s[e] += ss[e * 256 + q * C8 + cv];
        m[e] = fmaxf(m[e], sm[e * 256 + q * C8 + cv]);
      }
    }
    const long long o = ((long long)b * kPoolSplit + sp) * C + cv * 8;
#pragma unroll
    for (int e = 0; e < 8; ++e) { psum[o + e] = s[e]; pmax[o + e] = m[e]; }
  }
}
// gate[b,c] = sigmoid(mlp(avg) + mlp(max)), mlp = Linear(C,R) -> ReLU -> Linear(R,C); one block per image
__global__ void cbam_mlp_kernel(const float* __restrict__ psum, const float* __restrict__ pmax, int HW,
                                const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2,
                                const float* __restrict__ b2, float* __restrict__ gate, int C, int R) {
  extern __shared__ float sm[];  // avg[C] | max[C] | hid[2R]
  float* avg = sm;
  float* mx = sm + C;
  float* hid = sm + 2 * C;
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f, m = -CUDART_INF_F;
    for (int sp = 0; sp < kPoolSplit; ++sp) {
      s += psum[((long long)b * kPoolSplit + sp) * C + c];
      m = fmaxf(m, pmax[((long long)b * kPoolSplit + sp) * C + c]);
    }
    avg[c] = s / HW;
    mx[c] = m;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  for (int r = warp; r < 2 * R; r += nwarp) {  // one warp per hidden unit: coalesced weight rows
    const float* src = (r < R) ? avg : mx;
    const float* wr = w1 + (long long)(r % R) * C;
    float a = 0.f;
    for (int c = lane; c < C; c += 32) a += wr[c] * src[c];
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) hid[r] = fmaxf(a + b1[r % R], 0.f);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 2.f * b2[c];
    for (int r = 0; r < R; ++r) a += w2[(long long)c * R + r] * (hid[r] + hid[R + r]);
    gate[b * C + c] = sigmoidf_(a);
  }
}
// per pixel: max and mean over channels of x * gate -> stats [B,HW,2]; one warp per pixel, 8 channels per lane and load
__global__ void cbam_stats_kernel(const __half* __restrict__ x, const __half* __restrict__ x_lo, const float* __restrict__ gate,
                                  float* __restrict__ stats, int B, int HW, int C) {
  const long long pix = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (pix >= (long long)B * HW) return;
  const int b = (int)(pix / HW);
  const __half* p = x + pix * C;
  const __half* pl = x_lo + pix * C;
  const float* g = gate + b * C;
  float s = 0.f, m = -CUDART_INF_F;
  for (int c = lane * 8; c < C; c += 256) {
    float v[8], l[8];
    ld8(p + c, v);
    ld8(pl + c, l);
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] += l[e];
    const float4 g0 = *reinterpret_cast<const float4*>(g + c), g1 = *reinterpret_cast<const float4*>(g + c + 4);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float t = v[e] * gg[e];
      s += t;
      m = fmaxf(m, t);
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  }
  if (lane == 0) { stats[pix * 2] = m; stats[pix * 2 + 1] = s / C; }
}
// out = x + x * gate * sigmoid(conv7x7(stats))   (FeatureFusion: g + attention(g)); one warp per pixel.  x = x + x_lo on
// input, raw written as (hi, lo), relu as hi
__global__ void cbam_apply_split_kernel(const __half* __restrict__ x, const __half* __restrict__ x_lo,
                                        const float* __restrict__ gate, const float* __restrict__ stats,
                                        const float* __restrict__ ws, const float* __restrict__ bs,
                                        __half* __restrict__ raw, __half* __restrict__ raw_lo, __half* __restrict__ relu,
                                        int B, int H, int W, int C) {
  const long long pix = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (pix >= (long long)B * H * W) return;
  const int b = (int)(pix / ((long long)H * W));
  const int rem = (int)(pix - (long long)b * H * W);
  const int y = rem / W, xq = rem - y * W;
  float a = 0.f;
  for (int t = lane; t < 98; t += 32) {
    const int ch = t / 49, k = t % 49, dy = k / 7 - 3, dx = k % 7 - 3;
    const int yy = y + dy, xx = xq + dx;
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) a += ws[t] * stats[(((long long)b * H + yy) * W + xx) * 2 + ch];
  }
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  const float sg = sigmoidf_(a + bs[0]);
  const float* g = gate + b * C;
  for (int c = lane * 8; c < C; c += 256) {
    float v[8], l[8], o[8];
    ld8(x + pix * C + c, v);
    ld8(x_lo + pix * C + c, l);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float t = v[e] + l[e];
      o[e] = t + t * g[c + e] * sg;
    }
    st8_split(raw + pix * C + c, raw_lo + pix * C + c, o);
    if (relu) st8(relu + pix * C + c, o, true);
  }
}

// ---------------------------------------------------------------- key projection tail (modules.py:73-78)
// y fp32 [Q, ld] = [key(CK) | d(1) | e(CK)] -> key [Q,CK], shrinkage [Q] = d^2+1, selection [Q,CK] = sigmoid(e)
__global__ void key_tail_kernel(const float* __restrict__ y, int ld, int Q, int CK, int n_parts, long long part_stride,
                                float* __restrict__ key, float* __restrict__ shr, float* __restrict__ sel) {
  // y = n_parts fp32 partial sums (split-K of the key projection conv), added here in a fixed order with RN adds
  const long long total = (long long)Q * CK;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long q = i / CK;
    const int c = (int)(i - q * CK);
    const float* row = y + q * ld;
    float k = row[c], e = row[CK + 1 + c], d = (c == 0) ? row[CK] : 0.f;
    for (int p = 1; p < n_parts; ++p) {
      const float* rp = row + p * part_stride;
      k += rp[c];
      e += rp[CK + 1 + c];
      if (c == 0) d += rp[CK];
    }
    key[i] = k;
    sel[i] = sigmoidf_(e);
    if (c == 0) shr[q] = d * d + 1.f;
  }
}

// ---------------------------------------------------------------- split-K finish
// out = sum_p parts[p] (+ res + res_lo), written as fp16 (hi, lo) pairs raw and / or ReLU'd: completes a split-precision
// convolution whose K loop ran as several short accumulation chains (conv.cu, `ksplit`).  The partial sums are added
// with round-to-nearest fp32 adds in a fixed order; part 0 carries the bias.
__global__ void __launch_bounds__(256)
sum_parts_kernel(const float* __restrict__ parts, int n_parts, long long part_stride, const __half* __restrict__ res,
                 const __half* __restrict__ res_lo, __half* __restrict__ raw, __half* __restrict__ raw_lo,
                 __half* __restrict__ relu, __half* __restrict__ relu_lo, long long n8) {
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n8; i += (long long)gridDim.x * 256) {
    const long long off = i * 8;
    float v[8], t[8];
    const float4 a = *reinterpret_cast<const float4*>(parts + off), b = *reinterpret_cast<const float4*>(parts + off + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    for (int p = 1; p < n_parts; ++p) {
      const float* src = parts + p * part_stride + off;
      const float4 c = *reinterpret_cast<const float4*>(src), d = *reinterpret_cast<const float4*>(src + 4);
      v[0] += c.x; v[1] += c.y; v[2] += c.z; v[3] += c.w; v[4] += d.x; v[5] += d.y; v[6] += d.z; v[7] += d.w;
    }
    if (res) {
      ld8(res + off, t);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] += t[e];
    }
    if (res_lo) {
      ld8(res_lo + off, t);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] += t[e];
    }
    if (raw) {
      if (raw_lo) st8_split(raw + off, raw_lo + off, v);
      else st8(raw + off, v, false);
    }
    if (relu) {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = fmaxf(v[e], 0.f);
      if (relu_lo) st8_split(relu + off, relu_lo + off, v);
      else st8(relu + off, v, false);
    }
  }
}

// ---------------------------------------------------------------- output tail (network.py:33-40,144-168)
// logits fp32 [K,h,w] (pred output) -> aggregated log-odds [(K+1),h,w]
__global__ void aggregate_kernel(const float* __restrict__ logits, float* __restrict__ agg, int K, int HW) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= HW) return;
  float bg = 1.f;
  for (int k = 0; k < K; ++k) {
    const float pk = sigmoidf_(logits[(long long)k * HW + i]);
    bg *= (1.f - pk);
    const float c = fminf(fmaxf(pk, 1e-7f), 1.f - 1e-7f);
    agg[(long long)(k + 1) * HW + i] = logf(c / (1.f - c));
  }
  const float c = fminf(fmaxf(bg, 1e-7f), 1.f - 1e-7f);
  agg[i] = logf(c / (1.f - c));
}
// bilinear x4 (align_corners=False) of agg [(K+1),h,w] + softmax over channels -> prob (and logits) [(K+1),4h,4w]
__global__ void up4_softmax_kernel(const float* __restrict__ agg, float* __restrict__ prob, float* __restrict__ logits_out,
                                   int K1, int h, int w) {
  const int H = 4 * h, W = 4 * w;
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= (long long)H * W) return;
  const int Y = (int)(i / W), X = (int)(i - (long long)Y * W);
  const float sy = fmaxf((Y + 0.5f) * 0.25f - 0.5f, 0.f), sx = fmaxf((X + 0.5f) * 0.25f - 0.5f, 0.f);
  const int y0 = (int)sy, x0 = (int)sx;
  const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
  const float wy = sy - y0, wx = sx - x0;
  const long long o00 = (long long)y0 * w + x0, o01 = (long long)y0 * w + x1, o10 = (long long)y1 * w + x0,
                  o11 = (long long)y1 * w + x1;
  if (K1 <= 32) {  // the usual case: the K+1 interpolated logits stay in registers, prob is written once
    float v[32];
    float m = -CUDART_INF_F;
#pragma unroll
    for (int k = 0; k < 32; ++k) {
      if (k < K1) {
        const float* a = agg + (long long)k * h * w;
        const float top = a[o00] + (a[o01] - a[o00]) * wx, bot = a[o10] + (a[o11] - a[o10]) * wx;
        v[k] = top + (bot - top) * wy;
        if (logits_out) logits_out[(long long)k * H * W + i] = v[k];
        m = fmaxf(m, v[k]);
      }
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) {
      if (k < K1) {
        v[k] = expf(v[k] - m);
        s += v[k];
      }
    }
    const float inv = 1.f / s;
#pragma unroll
    for (int k = 0; k < 32; ++k)
      if (k < K1) prob[(long long)k * H * W + i] = v[k] * inv;
    return;
  }
  float m = -CUDART_INF_F;
  for (int k = 0; k < K1; ++k) {
    const float* a = agg + (long long)k * h * w;
    const float top = a[o00] + (a[o01] - a[o00]) * wx, bot = a[o10] + (a[o11] - a[o10]) * wx;
    const float v = top + (bot - top) * wy;
    prob[(long long)k * H * W + i] = v;  // stash the logit
    if (logits_out) logits_out[(long long)k * H * W + i] = v;
    m = fmaxf(m, v);
  }
  float s = 0.f;
  for (int k = 0; k < K1; ++k) {
    const float e = expf(prob[(long long)k * H * W + i] - m);
    prob[(long long)k * H * W + i] = e;
    s += e;
  }
  const float inv = 1.f / s;
  for (int k = 0; k < K1; ++k) prob[(long long)k * H * W + i] *= inv;
}

// 3x3 gather of the fused logit head: z fp32 [B,H,W,9] (z[..., t] = <relu(p4), w_t>) ->
// logits[b,y,x] = bias + sum_{t=(dy+1)*3+(dx+1)} z[b, y+dy, x+dx, t]  (zero padding)  == Conv2d(256,1,3,pad=1)
__global__ void head_gather3x3_kernel(const float* __restrict__ z, float* __restrict__ out, float bias, int B, int H, int W) {
  const long long total = (long long)B * H * W;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int x = (int)(i % W);
    long long p = i / W;
    const int y = (int)(p % H);
    const int b = (int)(p / H);
    float a = bias;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) a += z[(((long long)b * H + yy) * W + xx) * 9 + t];
    }
    out[i] = a;
  }
}

// fp16 token-major [n, C] -> fp16 bank rows dst[c, j] (ld_dst): value append from the NHWC encoder output
__global__ void transpose_append_kernel(const __half* __restrict__ src, __half* __restrict__ dst, long long ld_dst, int n,
                                        int C) {
  __shared__ __half tile[32][33];
  const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int r = ty; r < 32; r += 8)
    tile[r][tx] = (n0 + r < n && c0 + tx < C) ? src[(long long)(n0 + r) * C + c0 + tx] : __float2half_rn(0.f);
  __syncthreads();
  for (int r = ty; r < 32; r += 8)
    if (c0 + r < C && n0 + tx < n) dst[(long long)(c0 + r) * ld_dst + n0 + tx] = tile[tx][r];
}
// fp32 [rows, Q] channel-major (readout GEMM output) -> fp16 NHWC-style [Q, rows]... not needed: the readout GEMM
// writes token-major directly (see readout.cu).

}  // namespace ew

static int grid_of(long long total) {
  long long g = (total + 255) / 256;
  const long long cap = (long long)sm_count() * 32;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace b200

using namespace b200;

extern "C" {

DEVA_B200_API int deva_b200_nchw_to_nhwc(const float* src, void* dst, int b, int c, int h, int w, int c_pad,
                                         deva_stream_t stream) {
  ew::nchw_to_nhwc_kernel<<<grid_of((long long)b * h * w * c_pad), 256, 0, S(stream)>>>(src, H(dst), b, c, h, w, c_pad);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_stem_im2col(const float* src, void* dst, void* dst_lo, int b, int c, int h, int w, int k_pad,
                                        deva_stream_t stream) {
  B200_REQUIRE(h % 2 == 0 && w % 2 == 0 && k_pad % 64 == 0 && k_pad >= 49 * c, "stem_im2col: bad shape");
  B200_REQUIRE(c >= 1 && c <= 8, "stem_im2col: at most 8 input planes");
  __half* hi = H(dst);
  __half* lo = H(dst_lo);
  const cudaStream_t s = S(stream);
  const size_t smem = (size_t)c * 7 * (2 * ew::IM_XT + 5) * sizeof(float);
  // the network's shapes: one thread per output pixel, whole im2col rows written with 16-byte stores
  const dim3 gx(ceil_div(w / 2, ew::IM1_XT));
  if (c == 1 && k_pad == 64 && !lo) {
    ew::stem_im2col_px_kernel<1, 4, false><<<dim3(gx.x, b * ceil_div(h / 2, 4)), ew::IM1_XT, 0, s>>>(src, hi, nullptr, b, h, w);
    B200_LAUNCH_CHECK();
    return 0;
  }
  if (c == 3 && k_pad == 192) {
    if (lo) ew::stem_im2col_px_kernel<3, 2, true><<<dim3(gx.x, b * ceil_div(h / 2, 2)), ew::IM1_XT, 0, s>>>(src, hi, lo, b, h, w);
    else ew::stem_im2col_px_kernel<3, 2, false><<<dim3(gx.x, b * ceil_div(h / 2, 2)), ew::IM1_XT, 0, s>>>(src, hi, nullptr, b, h, w);
    B200_LAUNCH_CHECK();
    return 0;
  }
  ew::stem_im2col_kernel<<<dim3(ceil_div(w / 2, ew::IM_XT), b * (h / 2)), 256, smem, s>>>(src, hi, lo, b, c, h, w, k_pad);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_maxpool(const void* x, const void* x_lo, void* y, void* y_lo, int b, int h, int w, int c,
                                    deva_stream_t stream) {
  B200_REQUIRE(c % 8 == 0, "maxpool: C %% 8");
  ew::maxpool_kernel<<<grid_of((long long)b * ((h + 1) / 2) * ((w + 1) / 2) * (c / 8)), 256, 0, S(stream)>>>(
      H(x), H(x_lo), H(y), H(y_lo), b, h, w, c);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_up2_add_split(const void* g, const void* g_lo, const void* skip, const void* skip_lo,
                                          void* raw, void* raw_lo, void* relu, void* relu_lo8, int b, int h, int w, int c,
                                          deva_stream_t stream) {
  B200_REQUIRE(c % 8 == 0 && g_lo && skip_lo && raw && raw_lo && (!relu_lo8 || relu),
               "up2_add_split: C %% 8, g_lo, skip_lo, raw and raw_lo are required, and relu with relu_lo8");
  ew::up2_add_split_kernel<<<dim3(ceil_div((w + 1) * (c / 8), 256), b * (h + 1)), 256, 0, S(stream)>>>(
      H(g), H(g_lo), H(skip), H(skip_lo), H(raw), H(raw_lo), H(relu), reinterpret_cast<unsigned char*>(relu_lo8), b, h, w,
      c);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_area_down(const void* x, void* y, int b, int h, int w, int c, int r, deva_stream_t stream) {
  B200_REQUIRE(c % 8 == 0 && h % r == 0 && w % r == 0, "area_down: shape");
  ew::area_down_kernel<<<grid_of((long long)b * (h / r) * (w / r) * (c / 8)), 256, 0, S(stream)>>>(H(x), H(y), b, h, w, c, r);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_area_down_plane(const float* x, float* y, int b, int h, int w, int r, deva_stream_t stream) {
  B200_REQUIRE(h % r == 0 && w % r == 0, "area_down_plane: shape");
  ew::area_down_plane_kernel<<<grid_of((long long)b * (h / r) * (w / r)), 256, 0, S(stream)>>>(x, y, b, h, w, r);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_cbam_split(const void* x, const void* x_lo, const float* w1, const float* b1, const float* w2,
                                       const float* b2, const float* ws, const float* bs, float* scratch, void* raw,
                                       void* raw_lo, void* relu, int b, int h, int w, int c, int r, deva_stream_t stream) {
  // the gate statistics are pooled over x + x_lo as well: a gate error is common to every channel of a pixel, so it
  // does not average out in the next convolution the way independent roundings do
  B200_REQUIRE(x_lo && raw && raw_lo, "cbam_split: the hi/lo tensors are required");
  const __half* xh = H(x);
  const __half* xl = H(x_lo);
  const cudaStream_t s = S(stream);
  // scratch: psum[B*kPoolSplit*C] | pmax[B*kPoolSplit*C] | gate[B*C] | stats[B*H*W*2]
  float* psum = scratch;
  float* pmax = psum + (long long)b * ew::kPoolSplit * c;
  float* gate = pmax + (long long)b * ew::kPoolSplit * c;
  float* stats = gate + (long long)b * c;
  const int HW = h * w;
  B200_REQUIRE(c % 8 == 0 && c / 8 <= 256 && 256 % (c / 8) == 0, "cbam_split: C = %d must be 8 x a divisor of 256", c);
  ew::cbam_pool_kernel<<<dim3(b, ew::kPoolSplit), 256, 0, s>>>(xh, xl, psum, pmax, HW, c);
  B200_LAUNCH_CHECK();
  ew::cbam_mlp_kernel<<<b, 256, (2 * c + 2 * r) * sizeof(float), s>>>(psum, pmax, HW, w1, b1, w2, b2, gate, c, r);
  B200_LAUNCH_CHECK();
  const long long warps = (long long)b * HW;
  ew::cbam_stats_kernel<<<ceil_div(warps * 32, 256), 256, 0, s>>>(xh, xl, gate, stats, b, HW, c);
  B200_LAUNCH_CHECK();
  ew::cbam_apply_split_kernel<<<ceil_div(warps * 32, 256), 256, 0, s>>>(xh, xl, gate, stats, ws, bs, H(raw), H(raw_lo),
                                                                        H(relu), b, h, w, c);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_key_tail(const float* y, int ld, int q, int ck, int n_parts, int64_t part_stride, float* key,
                                     float* shrinkage, float* selection, deva_stream_t stream) {
  B200_REQUIRE(n_parts >= 1, "key_tail: n_parts %d", n_parts);
  ew::key_tail_kernel<<<grid_of((long long)q * ck), 256, 0, S(stream)>>>(y, ld, q, ck, n_parts, part_stride, key, shrinkage,
                                                                         selection);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_sum_parts(const float* parts, int n_parts, int64_t part_stride, const void* res,
                                      const void* res_lo, void* raw, void* raw_lo, void* relu, void* relu_lo, int64_t n,
                                      deva_stream_t stream) {
  B200_REQUIRE(n_parts >= 1 && n % 8 == 0 && part_stride % 4 == 0 && (raw || relu), "sum_parts: bad shape");
  ew::sum_parts_kernel<<<grid_of(n / 8), 256, 0, S(stream)>>>(parts, n_parts, part_stride, H(res), H(res_lo), H(raw),
                                                              H(raw_lo), H(relu), H(relu_lo), n / 8);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_output_tail(const float* logits, float* agg, float* prob, float* logits_out, int k, int h,
                                        int w, deva_stream_t stream) {
  const cudaStream_t s = S(stream);
  ew::aggregate_kernel<<<ceil_div(h * w, 256), 256, 0, s>>>(logits, agg, k, h * w);
  B200_LAUNCH_CHECK();
  ew::up4_softmax_kernel<<<ceil_div(16ll * h * w, 256), 256, 0, s>>>(agg, prob, logits_out, k + 1, h, w);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_head_gather3x3(const float* z, float* out, float bias, int b, int h, int w,
                                           deva_stream_t stream) {
  ew::head_gather3x3_kernel<<<grid_of((long long)b * h * w), 256, 0, S(stream)>>>(z, out, bias, b, h, w);
  B200_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"

// ---------------------------------------------------------------- frame ingest / egress (SURVEY 8f-3)
namespace b200 {
namespace ew {
// u8 [h, w, 3] -> fp32 [3, h, w]: ToTensor (x / 255) then Normalize ((x - mean) / std), IEEE divisions like torch
__global__ void __launch_bounds__(256)
ingest_rgb8_kernel(const unsigned char* __restrict__ src, float* __restrict__ dst, long long hw, float m0, float m1,
                   float m2, float s0, float s1, float s2) {
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= hw) return;
  const unsigned char* p = src + 3 * i;
  dst[i] = __fdiv_rn(__fdiv_rn((float)p[0], 255.f) - m0, s0);
  dst[hw + i] = __fdiv_rn(__fdiv_rn((float)p[1], 255.f) - m1, s1);
  dst[2 * hw + i] = __fdiv_rn(__fdiv_rn((float)p[2], 255.f) - m2, s2);
}

// Source taps of output pixel (oy, ox) of a bilinear resize (align_corners = False, PyTorch's upsample_bilinear2d
// arithmetic) of one [h, w] plane to [out_h, out_w]; the same for every channel, so computed once per pixel.
struct ResizeTaps {
  long long off;  // offset in the plane of the top-left source pixel (of the pixel itself when `same`)
  int dx, dy;     // offsets of the right / lower neighbour, 0 at the last column / row
  float lx0, lx1, ly0, ly1;
  bool same;      // out_h == h && out_w == w: the value is read, not interpolated
};
__device__ __forceinline__ ResizeTaps resize_taps(int h, int w, int out_h, int out_w, float rh, float rw, int oy, int ox) {
  ResizeTaps t;
  t.same = out_h == h && out_w == w;
  if (t.same) {
    t.off = (long long)oy * w + ox;
    t.dx = t.dy = 0;
    t.lx0 = t.ly0 = 1.f;
    t.lx1 = t.ly1 = 0.f;
    return t;
  }
  const float sy = fmaxf(rh * (oy + 0.5f) - 0.5f, 0.f), sx = fmaxf(rw * (ox + 0.5f) - 0.5f, 0.f);
  const int y0 = (int)sy, x0 = (int)sx;
  t.dx = x0 < w - 1 ? 1 : 0;
  t.dy = y0 < h - 1 ? w : 0;
  t.ly1 = sy - y0; t.ly0 = 1.f - t.ly1; t.lx1 = sx - x0; t.lx0 = 1.f - t.lx1;
  t.off = (long long)y0 * w + x0;
  return t;
}
// Value of one channel plane at the output pixel of `t`.  Every egress kernel reads its values through this one
// function, so their id maps and scores come from the same float, bit for bit.  A uint8 plane (bool or byte masks) is
// read as bytes and each tap converted to float, which is what resizing `masks.float()` computes.  For 0 / 1 masks the
// compiled form (source index fma(r, o + 0.5, -0.5), row blend fma(ly0, top, ly1 * bot)) makes the same > 0.5 decisions
// as torch's CPU resize, which segment_with_text's reference thresholds (tests/test_detector_masks_cpu.py).
template <typename T>
__device__ __forceinline__ float resized_value(const T* __restrict__ plane, const ResizeTaps& t) {
  const T* q = plane + t.off;
  if (t.same) return (float)q[0];
  return t.ly0 * (t.lx0 * (float)q[0] + t.lx1 * (float)q[t.dx]) +
         t.ly1 * (t.lx0 * (float)q[t.dy] + t.lx1 * (float)q[t.dy + t.dx]);
}

// Channel of the first maximum of prob [c, h, w] resized to [out_h, out_w], at output pixel (oy, ox); channels
// streamed.
__device__ __forceinline__ int resized_argmax(const float* __restrict__ prob, int c, int h, int w, int out_h, int out_w,
                                              float rh, float rw, int oy, int ox) {
  const ResizeTaps t = resize_taps(h, w, out_h, out_w, rh, rw, oy, ox);
  const long long plane = (long long)h * w;
  int best = 0;
  float best_v;
  if (t.same) {
    best_v = resized_value(prob, t);
    for (int k = 1; k < c; ++k) {
      const float v = resized_value(prob + k * plane, t);
      if (v > best_v) { best_v = v; best = k; }
    }
  } else {
    best_v = -INFINITY;
    for (int k = 0; k < c; ++k) {
      const float v = resized_value(prob + k * plane, t);
      if (v > best_v) { best_v = v; best = k; }
    }
  }
  return best;
}

// prob [c, h, w] -> ids [out_h, out_w]: bilinear resize, flip, argmax (first maximum), id remap.  One thread per output
// pixel.
__global__ void __launch_bounds__(256)
prob_to_ids_kernel(const float* __restrict__ prob, int c, int h, int w, int out_h, int out_w, int flip, float rh,
                   float rw, const int* __restrict__ lut, unsigned char* __restrict__ out_u8,
                   long long* __restrict__ out_i64) {
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= (long long)out_h * out_w) return;
  const int oy = (int)(i / out_w), ox_out = (int)(i - (long long)oy * out_w);
  const int ox = flip ? out_w - 1 - ox_out : ox_out;  // flip acts on the resized map
  const int best = resized_argmax(prob, c, h, w, out_h, out_w, rh, rw, oy, ox);
  const int id = lut ? lut[best] : best;
  if (out_u8) out_u8[i] = (unsigned char)id;
  if (out_i64) out_i64[i] = id;
}

// Score export of multi-scale / flip evaluation: prob [c, h, w] -> per channel s = (uint8)(v * 255) of the resized (and
// optionally flipped) value v, with one RN multiply and truncation: numpy's (x * 255).astype(np.uint8) on float32 for
// v in [0, 256 / 255).  Written to scores u8 [c, out_h, out_w] and / or added to the running sum int32 [c, out_h, out_w].
// One thread per output pixel, channels streamed; each thread owns its pixel in every plane, so the add needs no atomic.
__global__ void __launch_bounds__(256)
prob_to_scores_kernel(const float* __restrict__ prob, int c, int h, int w, int out_h, int out_w, int flip, float rh,
                      float rw, unsigned char* __restrict__ scores, int* __restrict__ sum) {
  const long long n = (long long)out_h * out_w;
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= n) return;
  const int oy = (int)(i / out_w), ox_out = (int)(i - (long long)oy * out_w);
  const int ox = flip ? out_w - 1 - ox_out : ox_out;  // flip acts on the resized map
  const ResizeTaps t = resize_taps(h, w, out_h, out_w, rh, rw, oy, ox);
  const long long plane = (long long)h * w;
  for (int k = 0; k < c; ++k) {
    const float v = resized_value(prob + k * plane, t);
    const unsigned s = __float2uint_rz(__fmul_rn(v, 255.f)) & 255u;
    if (scores) scores[k * n + i] = (unsigned char)s;
    if (sum) sum[k * n + i] += (int)s;
  }
}

// Merge of multi-scale / flip scores: sum int32 [c, n] -> channel of the first maximum (np.argmax's tie order), mapped
// through lut (or kept when lut is null).  One thread per pixel, channels streamed.
__global__ void __launch_bounds__(256)
scores_to_ids_kernel(const int* __restrict__ sum, int c, long long n, const int* __restrict__ lut,
                     unsigned char* __restrict__ out_u8, long long* __restrict__ out_i64) {
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= n) return;
  int best = 0, best_v = sum[i];
  for (int k = 1; k < c; ++k) {
    const int v = sum[k * n + i];
    if (v > best_v) { best_v = v; best = k; }
  }
  const int id = lut ? lut[best] : best;
  if (out_u8) out_u8[i] = (unsigned char)id;
  if (out_i64) out_i64[i] = id;
}

// prob_to_segments' shared-memory histogram takes 20 bytes per channel
constexpr int kMaxSegmentChannels = DEVA_B200_MAX_SEGMENT_CHANNELS;

// Result-saver egress: the same argmax as prob_to_ids_kernel, then per output pixel (each output optional)
//   index u8 = (uint8)lut[k]; id image = bytes of rgb[k] (id % 256, id / 256 % 256, id / 65536, or 0 when the id is not
//   coloured); overlay = frame where lut[k] == 0, else (frame + id image) >> 1.
// The overlay is the reference's float32 blend image * a + rgb * (1 - a), a = 1 where the id is 0 and 0.5 elsewhere,
// truncated to uint8: with a = 1 it is image * 1 + rgb * 0 = image; with a = 0.5 both halves of 8-bit integers and
// their sum are exact in float32, so the blend is (image + rgb) / 2 exactly and truncation is the floor.
// Per channel k, counts[k] (pixels whose argmax is k) and boxes[k] = (x_min, y_min, x_max, y_max) accumulate in shared
// memory (5 ints per channel) over a grid-stride loop, then merge into global memory with atomics.
__global__ void __launch_bounds__(256)
prob_to_segments_kernel(const float* __restrict__ prob, int c, int h, int w, int out_h, int out_w, float rh, float rw,
                        const int* __restrict__ lut, const unsigned* __restrict__ rgb,
                        const unsigned char* __restrict__ frame, unsigned char* __restrict__ out_u8,
                        unsigned char* __restrict__ out_rgb, unsigned char* __restrict__ out_overlay,
                        unsigned long long* __restrict__ counts, int* __restrict__ boxes) {
  extern __shared__ int stats[];  // [5][c]: count, x_min, y_min, x_max, y_max
  const bool with_stats = counts != nullptr;
  if (with_stats) {
    for (int k = threadIdx.x; k < c; k += 256) {
      stats[k] = 0;
      stats[c + k] = INT_MAX;
      stats[2 * c + k] = INT_MAX;
      stats[3 * c + k] = -1;
      stats[4 * c + k] = -1;
    }
    __syncthreads();
  }
  const long long n = (long long)out_h * out_w;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const int oy = (int)(i / out_w), ox = (int)(i - (long long)oy * out_w);
    const int k = resized_argmax(prob, c, h, w, out_h, out_w, rh, rw, oy, ox);
    if (out_u8) out_u8[i] = (unsigned char)lut[k];
    if (out_rgb || out_overlay) {
      const unsigned v = rgb[k];
      const unsigned char r = v & 255u, g = (v >> 8) & 255u, b = (v >> 16) & 255u;
      if (out_rgb) {
        out_rgb[3 * i] = r;
        out_rgb[3 * i + 1] = g;
        out_rgb[3 * i + 2] = b;
      }
      if (out_overlay) {
        const unsigned char* f = frame + 3 * i;
        const bool keep = lut[k] == 0;
        out_overlay[3 * i] = keep ? f[0] : (unsigned char)((f[0] + r) >> 1);
        out_overlay[3 * i + 1] = keep ? f[1] : (unsigned char)((f[1] + g) >> 1);
        out_overlay[3 * i + 2] = keep ? f[2] : (unsigned char)((f[2] + b) >> 1);
      }
    }
    if (with_stats) {
      atomicAdd(&stats[k], 1);
      atomicMin(&stats[c + k], ox);
      atomicMin(&stats[2 * c + k], oy);
      atomicMax(&stats[3 * c + k], ox);
      atomicMax(&stats[4 * c + k], oy);
    }
  }
  if (with_stats) {
    __syncthreads();
    for (int k = threadIdx.x; k < c; k += 256) {
      if (stats[k] == 0) continue;
      atomicAdd(&counts[k], (unsigned long long)stats[k]);
      atomicMin(&boxes[4 * k], stats[c + k]);
      atomicMin(&boxes[4 * k + 1], stats[2 * c + k]);
      atomicMax(&boxes[4 * k + 2], stats[3 * c + k]);
      atomicMax(&boxes[4 * k + 3], stats[4 * c + k]);
    }
  }
}

// counts = 0, boxes = (INT_MAX, INT_MAX, -1, -1): what an empty channel reports.
__global__ void __launch_bounds__(256)
segments_init_kernel(int c, unsigned long long* __restrict__ counts, int* __restrict__ boxes) {
  const int k = blockIdx.x * 256 + threadIdx.x;
  if (k >= c) return;
  counts[k] = 0;
  boxes[4 * k] = INT_MAX;
  boxes[4 * k + 1] = INT_MAX;
  boxes[4 * k + 2] = -1;
  boxes[4 * k + 3] = -1;
}

// Resized ingest, pass 1 (horizontal, the order torch's CPU separable resampler uses): u8 [h, w, 3] -> fp32 tmp
// [3, h, out_w].  Every source tap is normalised exactly like ingest_rgb8_kernel (through a 256-entry table per channel,
// same divisions), then tmp = sum_j x_w[ox, j] * v[y, x_idx[ox, j]] accumulated in ascending j with FMAs.
__global__ void __launch_bounds__(256)
resize_rows_rgb8_kernel(const unsigned char* __restrict__ src, int h, int w, int out_w, const int* __restrict__ x_idx,
                        const float* __restrict__ x_w, int taps, float* __restrict__ tmp, float m0, float m1, float m2,
                        float s0, float s1, float s2) {
  __shared__ float norm[3][256];
  for (int i = threadIdx.x; i < 768; i += 256) {
    const int c = i >> 8;
    const float m = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
    norm[c][i & 255] = __fdiv_rn(__fdiv_rn((float)(i & 255), 255.f) - m, sd);
  }
  __syncthreads();
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= (long long)h * out_w) return;
  const int y = (int)(i / out_w), ox = (int)(i - (long long)y * out_w);
  const unsigned char* row = src + (long long)y * w * 3;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (int j = 0; j < taps; ++j) {
    const unsigned char* p = row + 3 * x_idx[ox * taps + j];
    const float wt = x_w[ox * taps + j];
    a0 = __fmaf_rn(norm[0][p[0]], wt, a0);
    a1 = __fmaf_rn(norm[1][p[1]], wt, a1);
    a2 = __fmaf_rn(norm[2][p[2]], wt, a2);
  }
  const long long plane = (long long)h * out_w;
  tmp[i] = a0;
  tmp[plane + i] = a1;
  tmp[2 * plane + i] = a2;
}

// Resized ingest, pass 2 (vertical): tmp [3, h, out_w] -> dst [3, out_h, out_w], optionally flipped horizontally.
__global__ void __launch_bounds__(256)
resize_cols_kernel(const float* __restrict__ tmp, int h, int out_h, int out_w, const int* __restrict__ y_idx,
                   const float* __restrict__ y_w, int taps, int flip, float* __restrict__ dst) {
  const long long plane = (long long)out_h * out_w;
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= 3 * plane) return;
  const int c = (int)(i / plane);
  const long long r = i - c * plane;
  const int oy = (int)(r / out_w), ox = (int)(r - (long long)oy * out_w);
  const float* col = tmp + (long long)c * h * out_w + ox;
  float a = 0.f;
  for (int j = 0; j < taps; ++j) a = __fmaf_rn(col[(long long)y_idx[oy * taps + j] * out_w], y_w[oy * taps + j], a);
  dst[c * plane + (long long)oy * out_w + (flip ? out_w - 1 - ox : ox)] = a;
}

// Index mask u8 [h, w, C] -> Out [out_h, out_w] by row / column gather (nearest), optionally flipped after the resize.
// One channel is the index itself; three are an RGB id r + 256 g + 65536 b.
template <int C, typename Out>
__global__ void __launch_bounds__(256)
mask_gather_kernel(const unsigned char* __restrict__ src, int w, int out_h, int out_w, const int* __restrict__ x_idx,
                   const int* __restrict__ y_idx, int flip, Out* __restrict__ dst) {
  static_assert(C == 1 || C == 3, "one index or three RGB channels");
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= (long long)out_h * out_w) return;
  const int oy = (int)(i / out_w), ox = (int)(i - (long long)oy * out_w);
  const unsigned char* p = src + ((long long)y_idx[oy] * w + x_idx[flip ? out_w - 1 - ox : ox]) * C;
  if constexpr (C == 1) {
    dst[i] = p[0];
  } else {
    dst[i] = (Out)p[0] + 256 * (Out)p[1] + 65536 * (Out)p[2];
  }
}

// Pillow's 8-bit two-pass BILINEAR resample (libImaging Resample.c, ImagingResampleHorizontal_8bpc /
// ImagingResampleVertical_8bpc): per output pixel a window [lo, lo + n) of the input axis, 22-bit fixed-point
// coefficients, a half added before the sum and the result shifted back and clamped (clip8).
constexpr int kPilPrecision = 22;

__device__ __forceinline__ int pil_clip8(int ss) {
  ss >>= kPilPrecision;
  return ss < 0 ? 0 : (ss > 255 ? 255 : ss);
}
__device__ __forceinline__ void pil_store(unsigned char* p, int v) { *p = (unsigned char)v; }
// torch.FloatTensor(np.array(mask)) / 255: one correctly rounded float32 division
__device__ __forceinline__ void pil_store(float* p, int v) { *p = __fdiv_rn((float)v, 255.f); }

// Horizontal pass: src u8 [k, h, w] -> dst [k, h, out_w].  bounds int32 [out_w, 2] (first tap, taps), coef int32
// [out_w, taps].  Without bounds the axis keeps its size and the pass copies (the resize skips it).
template <typename Out>
__global__ void __launch_bounds__(256)
pil_resample_rows_kernel(const unsigned char* __restrict__ src, int k, int h, int w, int out_w,
                         const int* __restrict__ bounds, const int* __restrict__ coef, int taps, Out* __restrict__ dst) {
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= (long long)k * h * out_w) return;
  const long long row = i / out_w;
  const int ox = (int)(i - row * out_w);
  const unsigned char* s = src + row * w;
  if (!bounds) {
    pil_store(dst + i, s[ox]);
    return;
  }
  const int lo = bounds[2 * ox], n = bounds[2 * ox + 1];
  const int* c = coef + (long long)ox * taps;
  int ss = 1 << (kPilPrecision - 1);
  for (int j = 0; j < n; ++j) ss += (int)s[lo + j] * c[j];
  pil_store(dst + i, pil_clip8(ss));
}

// Vertical pass: src u8 [k, h, out_w] -> dst float [k, out_h, out_w] (v / 255), with the same tables along y.
__global__ void __launch_bounds__(256)
pil_resample_cols_kernel(const unsigned char* __restrict__ src, int k, int h, int out_h, int out_w,
                         const int* __restrict__ bounds, const int* __restrict__ coef, int taps, float* __restrict__ dst) {
  const long long plane = (long long)out_h * out_w;
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= k * plane) return;
  const int p = (int)(i / plane);
  const long long r = i - p * plane;
  const int oy = (int)(r / out_w), ox = (int)(r - (long long)oy * out_w);
  const int lo = bounds[2 * oy], n = bounds[2 * oy + 1];
  const int* c = coef + (long long)oy * taps;
  const unsigned char* s = src + (long long)p * h * out_w + ox;
  int ss = 1 << (kPilPrecision - 1);
  for (int j = 0; j < n; ++j) ss += (int)s[(long long)(lo + j) * out_w] * c[j];
  pil_store(dst + i, pil_clip8(ss));
}

// ---------------------------------------------------------------- detector masks -> detection id map
// (deva/ext/automatic_sam.py auto_segment, deva/ext/grounding_dino.py segment_with_text).  Masks are uint8 [n, h, w]
// (a bool tensor's bytes), resized to [out_h, out_w] on the fly through resize_taps / resized_value.
constexpr int kMaskStatsPix = 8192;  // output pixels per statistics block: fixes which pixels each partial sum holds
constexpr int kMaskSmemCounters = DEVA_B200_MASK_SMEM_COUNTERS;

// Statistics, pass 1: block (chunk p, mask k) sums the resized values of mask k over output pixels
// [p * kMaskStatsPix, (p + 1) * kMaskStatsPix) in a fixed order (per thread, then a fixed shared-memory tree) and counts
// those > 0.5.  The partial sums land in fixed slots, so a mask's area is the same float on every call.
__global__ void __launch_bounds__(256)
mask_stats_partial_kernel(const unsigned char* __restrict__ masks, int n_masks, int h, int w, int out_h, int out_w,
                          float rh, float rw, int chunks, float* __restrict__ part_area, int* __restrict__ part_cov) {
  __shared__ float ss[256];
  __shared__ int sc[256];
  const long long n = (long long)out_h * out_w, plane = (long long)h * w;
  const long long i0 = (long long)blockIdx.x * kMaskStatsPix, i1 = min(n, i0 + kMaskStatsPix);
  for (int k = blockIdx.y; k < n_masks; k += gridDim.y) {
    const unsigned char* m = masks + k * plane;
    float s = 0.f;
    int c = 0;
    for (long long i = i0 + threadIdx.x; i < i1; i += 256) {
      const int oy = (int)(i / out_w), ox = (int)(i - (long long)oy * out_w);
      const float v = resized_value(m, resize_taps(h, w, out_h, out_w, rh, rw, oy, ox));
      s += v;
      c += v > 0.5f;
    }
    ss[threadIdx.x] = s;
    sc[threadIdx.x] = c;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (threadIdx.x < o) {
        ss[threadIdx.x] += ss[threadIdx.x + o];
        sc[threadIdx.x] += sc[threadIdx.x + o];
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      part_area[(long long)k * chunks + blockIdx.x] = ss[0];
      part_cov[(long long)k * chunks + blockIdx.x] = sc[0];
    }
    __syncthreads();
  }
}
// Statistics, pass 2: area[k] = the partial sums of mask k added in chunk order; covered[k] likewise.
__global__ void __launch_bounds__(256)
mask_stats_reduce_kernel(const float* __restrict__ part_area, const int* __restrict__ part_cov, int n_masks, int chunks,
                         float* __restrict__ area, int* __restrict__ covered) {
  const int k = blockIdx.x * 256 + threadIdx.x;
  if (k >= n_masks) return;
  float s = 0.f;
  int c = 0;
  for (int p = 0; p < chunks; ++p) {
    s += part_area[(long long)k * chunks + p];
    c += part_cov[(long long)k * chunks + p];
  }
  if (area) area[k] = s;
  if (covered) covered[k] = c;
}

// Adds 1 to counter[key] for every active lane of the warp: one atomic per distinct key (the background slot is what
// most pixels of a block share).  key < 0 adds nothing.
__device__ __forceinline__ void warp_count(int* counter, int key) {
  const unsigned peers = __match_any_sync(__activemask(), key);
  if (key >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&counter[key], __popc(peers));
}

// Scored argmax: per output pixel the slot of the first maximum of [0.1, v_0 * s_0, ..., v_{n-1} * s_{n-1}] (slot 0 is
// the background, slot k + 1 mask k).  won[slot] counts the pixels each slot wins, kept[slot] those where the winner's
// own value is >= 0.5.  slot_out gets the winning slot, or with kept_only the winning slot where it is kept and 0
// elsewhere.  Counters in shared memory when 2 (n + 1) fit in kMaskSmemCounters, in global memory otherwise.
__global__ void __launch_bounds__(256)
mask_scored_argmax_kernel(const unsigned char* __restrict__ masks, int n_masks, int h, int w, int out_h, int out_w,
                          float rh, float rw, const float* __restrict__ score, int kept_only, int* __restrict__ slot_out,
                          int* __restrict__ won, int* __restrict__ kept, int smem_counters) {
  extern __shared__ int counters[];
  const int slots = n_masks + 1;
  int* cw = smem_counters ? counters : won;
  int* ck = smem_counters ? counters + slots : kept;
  if (smem_counters) {
    for (int k = threadIdx.x; k < 2 * slots; k += 256) counters[k] = 0;
    __syncthreads();
  }
  const long long n = (long long)out_h * out_w, plane = (long long)h * w;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const int oy = (int)(i / out_w), ox = (int)(i - (long long)oy * out_w);
    const ResizeTaps t = resize_taps(h, w, out_h, out_w, rh, rw, oy, ox);
    int best = 0;
    float best_s = 0.1f, best_v = 0.f;
    for (int k = 0; k < n_masks; ++k) {
      const float v = resized_value(masks + k * plane, t);
      const float s = __fmul_rn(v, __ldg(score + k));
      if (s > best_s) { best_s = s; best = k + 1; best_v = v; }
    }
    const bool keep = best > 0 && best_v >= 0.5f;
    slot_out[i] = (kept_only && !keep) ? 0 : best;
    warp_count(cw, best);
    warp_count(ck, keep ? best : -1);
  }
  if (smem_counters) {
    __syncthreads();
    for (int k = threadIdx.x; k < slots; k += 256) {
      if (counters[k]) atomicAdd(&won[k], counters[k]);
      if (counters[slots + k]) atomicAdd(&kept[k], counters[slots + k]);
    }
  }
}

// Last cover: per output pixel the slot (k + 1) of the last mask k in `order` whose resized value is > 0.5, 0 when
// none; covered[k] counts the pixels where mask k is > 0.5.  Counters as in mask_scored_argmax_kernel (n of them).
__global__ void __launch_bounds__(256)
mask_last_cover_kernel(const unsigned char* __restrict__ masks, int n_masks, int h, int w, int out_h, int out_w,
                       float rh, float rw, const int* __restrict__ order, int* __restrict__ slot_out,
                       int* __restrict__ covered, int smem_counters) {
  extern __shared__ int counters[];
  int* cc = smem_counters ? counters : covered;
  if (smem_counters) {
    for (int k = threadIdx.x; k < n_masks; k += 256) counters[k] = 0;
    __syncthreads();
  }
  const long long n = (long long)out_h * out_w, plane = (long long)h * w;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const int oy = (int)(i / out_w), ox = (int)(i - (long long)oy * out_w);
    const ResizeTaps t = resize_taps(h, w, out_h, out_w, rh, rw, oy, ox);
    const unsigned active = __activemask();
    int last = 0;
    for (int j = 0; j < n_masks; ++j) {
      const int k = __ldg(order + j);
      const bool on = resized_value(masks + k * plane, t) > 0.5f;
      const unsigned b = __ballot_sync(active, on);
      if (b && (threadIdx.x & 31) == __ffs(active) - 1) atomicAdd(&cc[k], __popc(b));
      if (on) last = k + 1;
    }
    slot_out[i] = last;
  }
  if (smem_counters) {
    __syncthreads();
    for (int k = threadIdx.x; k < n_masks; k += 256)
      if (counters[k]) atomicAdd(&covered[k], counters[k]);
  }
}
}  // namespace ew

}  // namespace b200

extern "C" {

DEVA_B200_API int deva_b200_ingest_rgb8(const uint8_t* src, float* dst, int h, int w, const float mean[3],
                                        const float stdv[3], deva_stream_t stream) {
  B200_REQUIRE(h > 0 && w > 0 && mean && stdv, "ingest_rgb8: bad arguments");
  const long long hw = (long long)h * w;
  ew::ingest_rgb8_kernel<<<(unsigned)ceil_div(hw, 256ll), 256, 0, S(stream)>>>(src, dst, hw, mean[0], mean[1], mean[2],
                                                                              stdv[0], stdv[1], stdv[2]);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_ingest_rgb8_resize(const uint8_t* src, int h, int w, int out_h, int out_w,
                                               const int32_t* x_idx, const float* x_w, int x_taps, const int32_t* y_idx,
                                               const float* y_w, int y_taps, float* scratch, float* dst, int flip,
                                               const float mean[3], const float stdv[3], deva_stream_t stream) {
  B200_REQUIRE(h > 0 && w > 0 && out_h > 0 && out_w > 0 && x_taps > 0 && y_taps > 0 && x_idx && x_w && y_idx && y_w &&
               scratch && mean && stdv, "ingest_rgb8_resize: bad arguments");
  const cudaStream_t s = S(stream);
  const long long n1 = (long long)h * out_w, n2 = 3ll * out_h * out_w;
  ew::resize_rows_rgb8_kernel<<<(unsigned)ceil_div(n1, 256ll), 256, 0, s>>>(src, h, w, out_w, x_idx, x_w, x_taps, scratch,
                                                                            mean[0], mean[1], mean[2], stdv[0], stdv[1],
                                                                            stdv[2]);
  B200_LAUNCH_CHECK();
  ew::resize_cols_kernel<<<(unsigned)ceil_div(n2, 256ll), 256, 0, s>>>(scratch, h, out_h, out_w, y_idx, y_w, y_taps, flip,
                                                                       dst);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_mask_nearest(const uint8_t* src, int h, int w, int out_h, int out_w, const int32_t* x_idx,
                                         const int32_t* y_idx, int flip, int64_t* dst, deva_stream_t stream) {
  B200_REQUIRE(h > 0 && w > 0 && out_h > 0 && out_w > 0 && x_idx && y_idx, "mask_nearest: bad arguments");
  const long long n = (long long)out_h * out_w;
  ew::mask_gather_kernel<1, long long><<<(unsigned)ceil_div(n, 256ll), 256, 0, S(stream)>>>(
      src, w, out_h, out_w, x_idx, y_idx, flip, reinterpret_cast<long long*>(dst));
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_mask_nearest_ids(const uint8_t* src, int channels, int h, int w, int out_h, int out_w,
                                             const int32_t* x_idx, const int32_t* y_idx, int flip, int32_t* dst,
                                             deva_stream_t stream) {
  B200_REQUIRE(src && dst && (channels == 1 || channels == 3) && h > 0 && w > 0 && out_h > 0 && out_w > 0 && x_idx &&
               y_idx, "mask_nearest_ids: bad arguments");
  const long long n = (long long)out_h * out_w;
  const unsigned blocks = (unsigned)ceil_div(n, 256ll);
  if (channels == 1)
    ew::mask_gather_kernel<1, int32_t><<<blocks, 256, 0, S(stream)>>>(src, w, out_h, out_w, x_idx, y_idx, flip, dst);
  else
    ew::mask_gather_kernel<3, int32_t><<<blocks, 256, 0, S(stream)>>>(src, w, out_h, out_w, x_idx, y_idx, flip, dst);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_pil_resample_u8(const uint8_t* src, int k, int h, int w, int out_h, int out_w,
                                            const int32_t* x_bounds, const int32_t* x_coef, int x_taps,
                                            const int32_t* y_bounds, const int32_t* y_coef, int y_taps, uint8_t* scratch,
                                            float* dst, deva_stream_t stream) {
  const bool horiz = out_w != w, vert = out_h != h;
  B200_REQUIRE(src && dst && k > 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0, "pil_resample_u8: bad arguments");
  B200_REQUIRE(!horiz || (x_bounds && x_coef && x_taps > 0), "pil_resample_u8: the horizontal pass needs its tables");
  B200_REQUIRE(!vert || (y_bounds && y_coef && y_taps > 0), "pil_resample_u8: the vertical pass needs its tables");
  B200_REQUIRE(!(horiz && vert) || scratch, "pil_resample_u8: two passes need the scratch plane");
  const cudaStream_t s = S(stream);
  const long long n1 = (long long)k * h * out_w, n2 = (long long)k * out_h * out_w;
  if (!vert) {  // one pass (or a copy) straight to float
    ew::pil_resample_rows_kernel<float><<<(unsigned)ceil_div(n1, 256ll), 256, 0, s>>>(
        src, k, h, w, out_w, horiz ? x_bounds : nullptr, x_coef, x_taps, dst);
    B200_LAUNCH_CHECK();
    return 0;
  }
  const uint8_t* mid = src;
  if (horiz) {
    ew::pil_resample_rows_kernel<unsigned char><<<(unsigned)ceil_div(n1, 256ll), 256, 0, s>>>(
        src, k, h, w, out_w, x_bounds, x_coef, x_taps, scratch);
    B200_LAUNCH_CHECK();
    mid = scratch;
  }
  ew::pil_resample_cols_kernel<<<(unsigned)ceil_div(n2, 256ll), 256, 0, s>>>(mid, k, h, out_h, out_w, y_bounds, y_coef,
                                                                             y_taps, dst);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_prob_to_ids(const float* prob, int c, int h, int w, int out_h, int out_w, int flip,
                                        const int32_t* lut, uint8_t* out_u8, int64_t* out_i64, deva_stream_t stream) {
  B200_REQUIRE(c >= 1 && h > 0 && w > 0 && out_h > 0 && out_w > 0 && (out_u8 || out_i64), "prob_to_ids: bad arguments");
  const long long n = (long long)out_h * out_w;
  ew::prob_to_ids_kernel<<<(unsigned)ceil_div(n, 256ll), 256, 0, S(stream)>>>(
      prob, c, h, w, out_h, out_w, flip, (float)h / out_h, (float)w / out_w, lut, out_u8,
      reinterpret_cast<long long*>(out_i64));
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_prob_to_scores(const float* prob, int c, int h, int w, int out_h, int out_w, int flip,
                                           uint8_t* scores, int32_t* sum, deva_stream_t stream) {
  B200_REQUIRE(prob && c >= 1 && h > 0 && w > 0 && out_h > 0 && out_w > 0 && (scores || sum),
               "prob_to_scores: bad arguments");
  const long long n = (long long)out_h * out_w;
  ew::prob_to_scores_kernel<<<(unsigned)ceil_div(n, 256ll), 256, 0, S(stream)>>>(prob, c, h, w, out_h, out_w, flip,
                                                                                 (float)h / out_h, (float)w / out_w, scores,
                                                                                 sum);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_scores_to_ids(const int32_t* sum, int c, int h, int w, const int32_t* lut, uint8_t* out_u8,
                                          int64_t* out_i64, deva_stream_t stream) {
  B200_REQUIRE(sum && c >= 1 && h > 0 && w > 0 && (out_u8 || out_i64), "scores_to_ids: bad arguments");
  const long long n = (long long)h * w;
  ew::scores_to_ids_kernel<<<(unsigned)ceil_div(n, 256ll), 256, 0, S(stream)>>>(sum, c, n, lut, out_u8,
                                                                               reinterpret_cast<long long*>(out_i64));
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_prob_to_segments(const float* prob, int c, int h, int w, int out_h, int out_w,
                                             const int32_t* lut, const uint32_t* rgb, const uint8_t* frame,
                                             uint8_t* out_u8, uint8_t* out_rgb, uint8_t* out_overlay, int64_t* counts,
                                             int32_t* boxes, deva_stream_t stream) {
  B200_REQUIRE(c >= 1 && h > 0 && w > 0 && out_h > 0 && out_w > 0 && lut, "prob_to_segments: bad arguments");
  B200_REQUIRE(c <= ew::kMaxSegmentChannels, "prob_to_segments: %d channels, at most %d supported", c,
               ew::kMaxSegmentChannels);
  B200_REQUIRE((!out_rgb && !out_overlay) || rgb, "prob_to_segments: the id image and overlay need the rgb table");
  B200_REQUIRE(!out_overlay || frame, "prob_to_segments: the overlay needs the frame");
  B200_REQUIRE(!counts == !boxes, "prob_to_segments: counts and boxes are written together");
  unsigned long long* counts_u64 = reinterpret_cast<unsigned long long*>(counts);
  const cudaStream_t s = S(stream);
  const long long n = (long long)out_h * out_w;
  long long blocks = (n + 255) / 256;
  size_t smem = 0;
  if (counts) {
    smem = 5ull * c * sizeof(int);
    blocks = std::min(blocks, 4ll * sm_count());  // fewer, longer-lived blocks amortise the per-block histogram
    B200_CUDA(cudaFuncSetAttribute(ew::prob_to_segments_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ew::segments_init_kernel<<<(unsigned)ceil_div(c, 256), 256, 0, s>>>(c, counts_u64, boxes);
    B200_LAUNCH_CHECK();
  }
  ew::prob_to_segments_kernel<<<(unsigned)blocks, 256, smem, s>>>(prob, c, h, w, out_h, out_w, (float)h / out_h,
                                                                   (float)w / out_w, lut, rgb, frame, out_u8, out_rgb,
                                                                   out_overlay, counts_u64, boxes);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API size_t deva_b200_mask_stats_workspace_bytes(int n, int out_h, int out_w) {
  const long long chunks = ((long long)out_h * out_w + ew::kMaskStatsPix - 1) / ew::kMaskStatsPix;
  return (size_t)(n < 0 ? 0 : n) * (size_t)chunks * (sizeof(float) + sizeof(int));
}
DEVA_B200_API int deva_b200_mask_stats(const uint8_t* masks, int n, int h, int w, int out_h, int out_w, void* workspace,
                                       float* area, int32_t* covered, deva_stream_t stream) {
  B200_REQUIRE(n >= 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0 && (n == 0 || (masks && workspace && (area || covered))),
               "mask_stats: bad arguments");
  if (n == 0) return 0;
  const cudaStream_t s = S(stream);
  const int chunks = ceil_div((long long)out_h * out_w, ew::kMaskStatsPix);
  float* part_area = reinterpret_cast<float*>(workspace);
  int* part_cov = reinterpret_cast<int*>(part_area + (long long)n * chunks);
  ew::mask_stats_partial_kernel<<<dim3(chunks, std::min(n, 65535)), 256, 0, s>>>(
      masks, n, h, w, out_h, out_w, (float)h / out_h, (float)w / out_w, chunks, part_area, part_cov);
  B200_LAUNCH_CHECK();
  ew::mask_stats_reduce_kernel<<<ceil_div(n, 256), 256, 0, s>>>(part_area, part_cov, n, chunks, area, covered);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_mask_scored_argmax(const uint8_t* masks, int n, int h, int w, int out_h, int out_w,
                                               const float* score, int kept_only, int32_t* slot, int32_t* won,
                                               int32_t* kept, deva_stream_t stream) {
  B200_REQUIRE(n >= 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0 && slot && won && kept && (n == 0 || (masks && score)),
               "mask_scored_argmax: bad arguments");
  const cudaStream_t s = S(stream);
  B200_CUDA(cudaMemsetAsync(won, 0, (n + 1) * sizeof(int32_t), s));
  B200_CUDA(cudaMemsetAsync(kept, 0, (n + 1) * sizeof(int32_t), s));
  const long long pixels = (long long)out_h * out_w;
  const bool smem = 2ll * (n + 1) <= ew::kMaskSmemCounters;
  // with shared counters, fewer and longer-lived blocks amortise zeroing and flushing them
  const long long blocks = smem ? std::min(ceil_div(pixels, 256), 4 * sm_count()) : ceil_div(pixels, 256);
  const size_t bytes = smem ? 2ull * (n + 1) * sizeof(int) : 0;  // at most 32 KiB: no opt-in needed
  ew::mask_scored_argmax_kernel<<<(unsigned)blocks, 256, bytes, s>>>(masks, n, h, w, out_h, out_w, (float)h / out_h,
                                                                      (float)w / out_w, score, kept_only, slot, won, kept,
                                                                      smem);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_mask_last_cover(const uint8_t* masks, int n, int h, int w, int out_h, int out_w,
                                            const int32_t* order, int32_t* slot, int32_t* covered,
                                            deva_stream_t stream) {
  B200_REQUIRE(n >= 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0 && slot && (n == 0 || (masks && order && covered)),
               "mask_last_cover: bad arguments");
  const cudaStream_t s = S(stream);
  if (n > 0) B200_CUDA(cudaMemsetAsync(covered, 0, n * sizeof(int32_t), s));
  const long long pixels = (long long)out_h * out_w;
  const bool smem = n <= ew::kMaskSmemCounters;
  const long long blocks = smem ? std::min(ceil_div(pixels, 256), 4 * sm_count()) : ceil_div(pixels, 256);
  const size_t bytes = smem ? (size_t)n * sizeof(int) : 0;
  ew::mask_last_cover_kernel<<<(unsigned)blocks, 256, bytes, s>>>(masks, n, h, w, out_h, out_w, (float)h / out_h,
                                                                   (float)w / out_w, order, slot, covered, smem);
  B200_LAUNCH_CHECK();
  return 0;
}
DEVA_B200_API int deva_b200_transpose_append(const void* src, void* dst, int64_t ld_dst, int n, int c,
                                             deva_stream_t stream) {
  ew::transpose_append_kernel<<<dim3(ceil_div(n, 32), ceil_div(c, 32)), 256, 0, S(stream)>>>(H(src), H(dst), ld_dst, n, c);
  B200_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
