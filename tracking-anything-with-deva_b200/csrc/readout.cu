// Memory readout  out[K*CV, Q] = V[K*CV, N] . P[N, Q]   (reference: MemoryManager._readout,
// deva/inference/memory_manager.py:64-75; training twin memory_utils.py:87-94).
//
// wgmma GEMM, fp16 operands / fp32 accumulation in registers.
//   A operand = value bank rows (M = value channels of the active objects), K-major: the bank
//               keeps every value row contiguous along the memory-slot axis N.
//   B operand = dense affinity P stored [Q, N] (K-major), produced by the top-k/softmax stage.
//   D         = 128 x 256 fp32 tile per CTA: two consumer warpgroups, 64 rows each (m64n256k16).
// Warp roles: warps 0-7 consumers (MMA + epilogue), warp 8 TMA producer.
// Persistent CTAs (one per SM) walk a grouped raster of the tile grid so that CTAs running
// together share value panels and affinity panels in L2.
#include <cuda_fp16.h>

#include <stdlib.h>

#include "common.h"
#include "ptx.cuh"
#include "tmap.h"

namespace b200 {
namespace readout {

constexpr int BM = 128, BN = 256, BK = 64;
constexpr int STAGES = 4;
constexpr int A_BYTES = BM * BK * 2;
constexpr int B_BYTES = BN * BK * 2;
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int CONSUMER_THREADS = 256;
constexpr int THREADS = CONSUMER_THREADS + 32;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
constexpr int GROUP_M = 16;
constexpr int kMaxGroups = DEVA_B200_MAX_GROUPS;  // objects per launch
constexpr int kMaxPeers = 8;  // ranks of one NVLink box (scatter-reduce mode)

struct Params {
  int m_tiles, n_tiles, k_blocks, tiles_per_group;
  int q;
  long long ldo;
  float* out;
  __half* out_tok;  // optional fp16 token-major output [object, q, rows_per_group]
  int rows_per_group;
  int val_row[kMaxGroups];
  int out_row[kMaxGroups];
};

__device__ __forceinline__ void tile_coords(int tile, int m_tiles, int n_tiles, int& m, int& n) {
  const int per_band = GROUP_M * n_tiles;
  const int band = tile / per_band;
  const int first_m = band * GROUP_M;
  const int rows = min(GROUP_M, m_tiles - first_m);
  const int r = tile - band * per_band;
  m = first_m + r % rows;
  n = r / rows;
}

// Consumer side of one tile: the k-loop over the shared-memory ring (a stage is released once the wgmma that read it
// have completed), leaving this warpgroup's 64 x BN accumulator in d.
__device__ __forceinline__ void mma_tile(float (&d)[BN / 2], const uint8_t* sA, const uint8_t* sB, uint64_t* full,
                                         uint64_t* empty, int k_blocks, int& stage, uint32_t& phase) {
  const uint32_t a_off = (threadIdx.x >> 7) * 64 * 128;  // this warpgroup's 64 rows of the A tile
  int prev = -1;
  for (int kb = 0; kb < k_blocks; ++kb) {
    mbar_wait(&full[stage], phase);
    const uint32_t a_addr = smem_u32(sA + stage * A_BYTES) + a_off;
    const uint32_t b_addr = smem_u32(sB + stage * B_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)
      wgmma_f16<BN>(d, wgmma_desc_sw128(a_addr + k * 32), wgmma_desc_sw128(b_addr + k * 32), (kb | k) != 0);
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(d);
  if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
}

// Row i (0: lane/4, 1: lane/4 + 8) of this thread's accumulator fragment -> fp32 row `dst` (columns q0 + 8j, +1), or
// the fp16 token-major output `dt` when given.
template <int W>
__device__ __forceinline__ void store_rows(const float (&d)[W / 2], int i, int q0, int q, float* dst, __half* dt,
                                           int rows_per_group, bool vec_ok) {
  if (dt) {
#pragma unroll
    for (int j = 0; j < W / 8; ++j) {
      const int c = q0 + 8 * j;
      if (c < q) dt[(long long)c * rows_per_group] = __float2half_rn(d[4 * j + 2 * i]);
      if (c + 1 < q) dt[(long long)(c + 1) * rows_per_group] = __float2half_rn(d[4 * j + 2 * i + 1]);
    }
  } else {
#pragma unroll
    for (int j = 0; j < W / 8; ++j) {
      const int c = q0 + 8 * j;
      if (vec_ok && c + 1 < q) {
        *reinterpret_cast<float2*>(dst + c) = make_float2(d[4 * j + 2 * i], d[4 * j + 2 * i + 1]);
      } else {
        if (c < q) dst[c] = d[4 * j + 2 * i];
        if (c + 1 < q) dst[c + 1] = d[4 * j + 2 * i + 1];
      }
    }
  }
}

__global__ void __launch_bounds__(THREADS, 1)
readout_kernel(const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_p,
               const __grid_constant__ Params p) {
  // 1024-byte alignment (128B swizzle atoms) comes from the declaration: deriving an aligned pointer through an
  // integer cast would make the compiler lose the shared address space (generic LD/ST instead of LDS/STS).
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full = bars;                 // [STAGES]
  uint64_t* empty = bars + STAGES;       // [STAGES]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int total_tiles = p.m_tiles * p.n_tiles;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&map_v);
    tma_prefetch_desc(&map_p);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int m, n;
        tile_coords(tile, p.m_tiles, p.n_tiles, m, n);
        const int g = m / p.tiles_per_group;
        const int a_row = p.val_row[g] + (m - g * p.tiles_per_group) * BM;
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], STAGE_BYTES);
          tma_load_2d(sA + stage * A_BYTES, &map_v, &full[stage], kb * BK, a_row);
          tma_load_2d(sB + stage * B_BYTES, &map_p, &full[stage], kb * BK, n * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  const bool vec_ok = (p.ldo % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 7) == 0);
  const int qd = lane & 3;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int m, n;
    tile_coords(tile, p.m_tiles, p.n_tiles, m, n);
    float d[BN / 2];
    mma_tile(d, sA, sB, full, empty, p.k_blocks, stage, phase);
    const int g = m / p.tiles_per_group;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
      const long long R = p.out_row[g] + (long long)(m - g * p.tiles_per_group) * BM + row;
      float* dst = p.out + R * p.ldo;
      __half* dt = nullptr;
      if (p.out_tok) {
        const long long obj = R / p.rows_per_group;
        dt = p.out_tok + (obj * p.q) * p.rows_per_group + (R - obj * p.rows_per_group);
      }
      store_rows<BN>(d, i, n * BN + 2 * qd, p.q, dst, dt, p.rows_per_group, vec_ok);
    }
  }
}


// ======================================================================================================
// Fused sparse-affinity readout.  The affinity has top_k non-zeros per query, so instead of reading a
// dense [Q, N] fp16 operand from HBM/L2 the B tile (256 queries x 64 slots, 128B-swizzled K-major) is BUILT IN
// SHARED MEMORY from the top-k lists: stage buffers are zeroed once, a generator warp scatters the ~50 non-zero
// weights of the current k-block, and clears exactly those again when the stage is recycled.  Only the value
// operand streams through TMA (16 KB instead of 48 KB per k-iteration), and no dense affinity is ever written.
// The lists (rows of ld_list entries: 32 for deva_b200_sim_topk's, wider for the wide read) are pre-bucketed per
// (256-query tile, 64-slot k-block) by bucket_kernel.
// ======================================================================================================
constexpr int SP_THREADS = CONSUMER_THREADS + 128;  // warps: 0-7 consumers, 8-11 value TMA + affinity generators (one per stage)
constexpr int SP_REC = 1024;      // per-stage record of scattered offsets (falls back to a full clear beyond)
constexpr int SP_SMEM = STAGES * STAGE_BYTES + 1024 + 256 + STAGES * SP_REC * 2;

// entry = (query_local << 24) | (slot_local << 16) | fp16 weight bits
__global__ void __launch_bounds__(256)
bucket_kernel(const int* __restrict__ idx, const float* __restrict__ w, int ld_list, int q, int top_k, int k_blocks,
              int* __restrict__ offsets, uint32_t* __restrict__ entries) {
  extern __shared__ int hist[];  // [k_blocks + 1]
  const int tile = blockIdx.x;
  const int q0 = tile * BN;
  const int nq = min(BN, q - q0);
  int* off = offsets + (long long)tile * (k_blocks + 1);
  uint32_t* ent = entries + (long long)tile * BN * ld_list;
  for (int i = threadIdx.x; i <= k_blocks; i += 256) hist[i] = 0;
  __syncthreads();
  const int total = nq * top_k;
  for (int i = threadIdx.x; i < total; i += 256) {
    const int ql = i / top_k, j = i - ql * top_k;
    const long long e = (long long)(q0 + ql) * ld_list + j;
    if (w[e] != 0.f) atomicAdd(&hist[idx[e] / BK + 1], 1);  // zero-weight entries (padding, other shards' slots) are dropped
  }
  __syncthreads();
  if (threadIdx.x == 0) {  // k_blocks is small (N/64): serial scan is fine
    int run = 0;
    for (int i = 0; i <= k_blocks; ++i) { run += hist[i]; hist[i] = run; off[i] = run; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < total; i += 256) {
    const int ql = i / top_k, j = i - ql * top_k;
    const long long e = (long long)(q0 + ql) * ld_list + j;
    if (w[e] == 0.f) continue;
    const int n = idx[e];
    const int kb = n / BK;
    const int pos = atomicAdd(&hist[kb], 1);
    const uint32_t hw = __half_as_ushort(__float2half_rn(w[e]));
    ent[pos] = ((uint32_t)ql << 24) | ((uint32_t)(n - kb * BK) << 16) | hw;
  }
}

struct SpParams {
  int m_tiles, n_tiles, k_blocks, tiles_per_group;
  int q;
  long long ldo;
  float* out;
  __half* out_tok;
  int rows_per_group;
  const int* offsets;        // [n_tiles][k_blocks + 1]
  const uint32_t* entries;   // [n_tiles][BN * ld_list]
  int ld_list;
  int val_row[kMaxGroups];
  int out_row[kMaxGroups];
  // scatter-reduce mode (bank-sharded read): group g's tile is ADDED (red.add over NVLink / locally) into the buffer
  // of the rank that owns the object, rank_dst[owner[g]] + out_row[g] * ldo, instead of stored to `out`
  float* rank_dst[kMaxPeers];
  unsigned char owner[kMaxGroups];
  bool reduce;
};

// Raise the stage's expected transaction bytes without arriving (the arrive follows once the affinity tile is built).
__device__ __forceinline__ void mbar_expect_tx_only(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void red_add_v2_sys(float* addr, float a, float b) {
  asm volatile("red.relaxed.sys.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

__global__ void __launch_bounds__(SP_THREADS, 1)
readout_sparse_kernel(const __grid_constant__ CUtensorMap map_v, const __grid_constant__ SpParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  uint16_t* rec = reinterpret_cast<uint16_t*>(smem + STAGES * STAGE_BYTES + 256);   // [STAGES][SP_REC] byte offsets / 2

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int total_tiles = p.m_tiles * p.n_tiles;

  // zero the affinity stage buffers once
  for (int i = threadIdx.x; i < STAGES * B_BYTES / 16; i += SP_THREADS)
    reinterpret_cast<uint4*>(sB)[i] = make_uint4(0, 0, 0, 0);
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&map_v);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);   // the stage's generator, after its scatter (the value tile completes as tx bytes)
      mbar_init(&empty[i], 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  fence_proxy_async();
  __syncthreads();

  if (warp >= 8) {
    // ---- warp 8+s owns pipeline stage s (k-iterations f = s, s+4, ...): it loads the value tile by TMA and builds the
    // affinity tile, so the ~2 dependent global loads per k-block (bucket offsets, entries) have four MMA periods to
    // complete ----
    const int stage = warp - 8;
    uint8_t* tileB = sB + stage * B_BYTES;
    uint16_t* r = rec + stage * SP_REC;
    const int my_tiles = (total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const long long total_iters = (long long)my_tiles * p.k_blocks;
    int prev = 0;
    for (long long f = stage; f < total_iters; f += STAGES) {
      const int lt = (int)(f / p.k_blocks), kb = (int)(f - (long long)lt * p.k_blocks);
      const int tile = blockIdx.x + lt * gridDim.x;
      int m, n;
      tile_coords(tile, p.m_tiles, p.n_tiles, m, n);
      const int* off = p.offsets + (long long)n * (p.k_blocks + 1);
      const uint32_t* ent = p.entries + (long long)n * BN * p.ld_list;
      const int e0 = off[kb], cnt = off[kb + 1] - e0;
      uint32_t e_a = 0, e_b = 0;   // first 64 entries prefetched before the stage is free
      if (lane < cnt) e_a = ent[e0 + lane];
      if (lane + 32 < cnt) e_b = ent[e0 + 32 + lane];
      mbar_wait(&empty[stage], (uint32_t)((f / STAGES) & 1) ^ 1u);
      if (lane == 0) {
        const int g = m / p.tiles_per_group;
        mbar_expect_tx_only(&full[stage], A_BYTES);
        tma_load_2d(sA + stage * A_BYTES, &map_v, &full[stage], kb * BK, p.val_row[g] + (m - g * p.tiles_per_group) * BM);
      }
      // clear what the previous use of this stage scattered
      if (prev > SP_REC) {
        for (int i = lane; i < B_BYTES / 16; i += 32) reinterpret_cast<uint4*>(tileB)[i] = make_uint4(0, 0, 0, 0);
      } else {
        for (int i = lane; i < prev; i += 32) reinterpret_cast<__half*>(tileB)[r[i]] = __ushort_as_half(0);
      }
      __syncwarp();
      for (int i = lane; i < cnt; i += 32) {
        const uint32_t e = (i < 32) ? e_a : ((i < 64) ? e_b : ent[e0 + i]);
        const uint32_t ql = e >> 24, sl = (e >> 16) & 63u;
        // K-major, 128-byte swizzle: row ql, 16-byte chunk (sl/8) XOR (ql%8), element sl%8 within the chunk
        const uint32_t hoff = ql * 64u + ((((sl >> 3) ^ (ql & 7u)) << 3) | (sl & 7u));
        reinterpret_cast<__half*>(tileB)[hoff] = __ushort_as_half((unsigned short)(e & 0xffffu));
        if (i < SP_REC) r[i] = (uint16_t)hoff;
      }
      prev = cnt;
      fence_proxy_async();   // generic-proxy smem writes -> visible to the tensor core (async proxy)
      __syncwarp();
      if (lane == 0) mbar_arrive(&full[stage]);
    }
  } else {
    const bool vec_ok = (p.ldo % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 7) == 0);
    const int qd = lane & 3;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int m, n;
      tile_coords(tile, p.m_tiles, p.n_tiles, m, n);
      float d[BN / 2];
      mma_tile(d, sA, sB, full, empty, p.k_blocks, stage, phase);
      const int g = m / p.tiles_per_group;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
        const long long R = p.out_row[g] + (long long)(m - g * p.tiles_per_group) * BM + row;
        float* dst = (p.reduce ? p.rank_dst[p.owner[g]] : p.out) + R * p.ldo;
        const long long obj = R / p.rows_per_group;
        __half* dt = p.out_tok ? p.out_tok + (obj * p.q) * p.rows_per_group + (R - obj * p.rows_per_group) : nullptr;
        if (p.reduce) {  // partial sums of this rank's slots -> the owner's buffer (peer memory or local)
          const bool vec = p.ldo % 2 == 0;  // 8-byte vector reductions need 8-byte aligned rows
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int q = n * BN + 8 * j + 2 * qd;
            if (vec && q + 1 < p.q) {
              red_add_v2_sys(dst + q, d[4 * j + 2 * i], d[4 * j + 2 * i + 1]);
            } else {
              if (q < p.q) atomicAdd_system(dst + q, d[4 * j + 2 * i]);
              if (q + 1 < p.q) atomicAdd_system(dst + q + 1, d[4 * j + 2 * i + 1]);
            }
          }
        } else {
          store_rows<BN>(d, i, n * BN + 2 * qd, p.q, dst, dt, p.rows_per_group, vec_ok);
        }
      }
    }
  }
}

}  // namespace readout
}  // namespace b200

using namespace b200;

extern "C" {

DEVA_B200_API int deva_b200_readout(const void* values, int64_t values_ld, int64_t values_rows, const int32_t* val_row,
                                    const int32_t* out_row, int n_groups, int rows_per_group, const void* affinity,
                                    int64_t ld_affinity, int n_window, int q, float* out, int64_t ld_out, void* out_tok,
                                    deva_stream_t stream) {
  using namespace readout;
  B200_REQUIRE(n_groups >= 1 && n_groups <= kMaxGroups, "readout: n_groups %d out of range [1,%d]", n_groups,
               kMaxGroups);
  B200_REQUIRE(rows_per_group % BM == 0, "readout: rows_per_group %d must be a multiple of %d", rows_per_group, BM);
  B200_REQUIRE(n_window >= 1 && q >= 1, "readout: empty problem");
  B200_REQUIRE(values_ld % 8 == 0 && ld_affinity % 8 == 0, "readout: leading dimensions must be multiples of 8 halves");
  const char* err = nullptr;
  CUtensorMap map_v, map_p;
  if (make_tmap_2d(&map_v, TmapType::F16, values, n_window, values_rows, values_ld * 2, BK, BM, &err) ||
      make_tmap_2d(&map_p, TmapType::F16, affinity, n_window, q, ld_affinity * 2, BK, BN, &err)) {
    set_error("readout: %s", err ? err : "tensor map");
    return 3;
  }
  Params p;
  p.tiles_per_group = rows_per_group / BM;
  p.m_tiles = n_groups * p.tiles_per_group;
  p.n_tiles = ceil_div(q, BN);
  p.k_blocks = ceil_div(n_window, BK);
  p.q = q;
  p.ldo = ld_out;
  p.out = out;
  p.out_tok = H(out_tok);
  p.rows_per_group = rows_per_group;
  for (int i = 0; i < n_groups; ++i) {
    p.val_row[i] = val_row[i];
    p.out_row[i] = out_row[i];
  }
  static bool configured_dev[kMaxDevices] = {false};  // function attributes are per device
  bool& configured = configured_dev[device_slot()];
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(readout_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    configured = true;
  }
  const int total = p.m_tiles * p.n_tiles;
  const int grid = total < sm_count() ? total : sm_count();
  readout_kernel<<<grid, THREADS, SMEM_BYTES, S(stream)>>>(map_v, map_p, p);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API size_t deva_b200_readout_sparse_wide_workspace_bytes(int q, int n_window, int ld_list) {
  const size_t n_tiles = (q + readout::BN - 1) / readout::BN;
  const size_t k_blocks = (n_window + readout::BK - 1) / readout::BK;
  return n_tiles * ((k_blocks + 1) * 4 + (size_t)readout::BN * ld_list * 4) + 256;
}

DEVA_B200_API size_t deva_b200_readout_sparse_workspace_bytes(int q, int n_window) {
  return deva_b200_readout_sparse_wide_workspace_bytes(q, n_window, kListCap);
}

}  // extern "C"

// The plain and the scatter-reduce sparse read-out (rank_dst given: group g's tile is red.add'ed into
// rank_dst[owner[g]] + out_row[g] * ld_out instead of stored to `out`).
static int readout_sparse(const void* values, int64_t values_ld, int64_t values_rows, const int32_t* val_row,
                          const int32_t* out_row, const int32_t* owner, int n_groups, int rows_per_group,
                          const int32_t* idx, const float* w, int ld_list, int top_k, int n_window, int q,
                          void* workspace, float* out,
                          float* const* rank_dst, int n_ranks, int64_t ld_out, void* out_tok, deva_stream_t stream) {
  using namespace readout;
  const cudaStream_t s = S(stream);
  B200_REQUIRE(!rank_dst || (owner && n_ranks >= 1 && n_ranks <= kMaxPeers && !out_tok),
               "readout: scatter-reduce needs owners and 1..%d destination ranks", kMaxPeers);
  B200_REQUIRE(n_groups >= 1 && n_groups <= kMaxGroups, "readout: n_groups %d out of range [1,%d]", n_groups, kMaxGroups);
  B200_REQUIRE(rows_per_group % BM == 0, "readout: rows_per_group %d must be a multiple of %d", rows_per_group, BM);
  B200_REQUIRE(n_window >= 1 && q >= 1 && top_k >= 1 && top_k <= ld_list && ld_list % 32 == 0, "readout: bad shape");
  B200_REQUIRE(values_ld % 8 == 0, "readout: leading dimension must be a multiple of 8 halves");
  const char* err = nullptr;
  CUtensorMap map_v;
  if (make_tmap_2d(&map_v, TmapType::F16, values, n_window, values_rows, values_ld * 2, BK, BM, &err)) {
    set_error("readout: %s", err ? err : "tensor map");
    return 3;
  }
  SpParams p;
  p.tiles_per_group = rows_per_group / BM;
  p.m_tiles = n_groups * p.tiles_per_group;
  p.n_tiles = ceil_div(q, BN);
  p.k_blocks = ceil_div(n_window, BK);
  p.q = q; p.ldo = ld_out; p.out = out; p.out_tok = H(out_tok); p.rows_per_group = rows_per_group;
  int* offsets = reinterpret_cast<int*>(workspace);
  uint32_t* entries = reinterpret_cast<uint32_t*>(offsets + (size_t)p.n_tiles * (p.k_blocks + 1));
  p.offsets = offsets; p.entries = entries; p.ld_list = ld_list;
  for (int i = 0; i < n_groups; ++i) { p.val_row[i] = val_row[i]; p.out_row[i] = out_row[i]; }
  p.reduce = rank_dst != nullptr;
  if (rank_dst) {
    for (int r = 0; r < n_ranks; ++r) p.rank_dst[r] = rank_dst[r];
    for (int i = 0; i < n_groups; ++i) {
      B200_REQUIRE(owner[i] >= 0 && owner[i] < n_ranks, "readout: owner %d out of range", owner[i]);
      p.owner[i] = (unsigned char)owner[i];
    }
  }
  B200_REQUIRE((size_t)(p.k_blocks + 1) * 4 <= 200 * 1024, "readout: window of %d slots too large for the bucket pass", n_window);
  static bool configured_dev[kMaxDevices] = {false};  // function attributes are per device
  bool& configured = configured_dev[device_slot()];
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(readout_sparse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SP_SMEM));
    B200_CUDA(cudaFuncSetAttribute(bucket_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  bucket_kernel<<<p.n_tiles, 256, (p.k_blocks + 1) * sizeof(int), s>>>(idx, w, ld_list, q, top_k, p.k_blocks, offsets,
                                                                        entries);
  B200_LAUNCH_CHECK();
  const int total = p.m_tiles * p.n_tiles;
  const int grid = total < sm_count() ? total : sm_count();
  readout_sparse_kernel<<<grid, SP_THREADS, SP_SMEM, s>>>(map_v, p);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" {

DEVA_B200_API int deva_b200_readout_sparse(const void* values, int64_t values_ld, int64_t values_rows,
                                           const int32_t* val_row, const int32_t* out_row, int n_groups,
                                           int rows_per_group, const int32_t* idx, const float* w, int top_k,
                                           int n_window, int q, void* workspace, float* out, int64_t ld_out,
                                           void* out_tok, deva_stream_t stream) {
  return readout_sparse(values, values_ld, values_rows, val_row, out_row, nullptr, n_groups, rows_per_group, idx, w,
                        kListCap, top_k, n_window, q, workspace, out, nullptr, 0, ld_out, out_tok, stream);
}

DEVA_B200_API int deva_b200_readout_sparse_scatter(const void* values, int64_t values_ld, int64_t values_rows,
                                                   const int32_t* val_row, const int32_t* out_row,
                                                   const int32_t* owner, int n_groups, int rows_per_group,
                                                   const int32_t* idx, const float* w, int top_k, int n_window, int q,
                                                   void* workspace, float* const* rank_dst, int n_ranks,
                                                   int64_t ld_out, deva_stream_t stream) {
  return readout_sparse(values, values_ld, values_rows, val_row, out_row, owner, n_groups, rows_per_group, idx, w,
                        kListCap, top_k, n_window, q, workspace, nullptr, rank_dst, n_ranks, ld_out, nullptr, stream);
}

DEVA_B200_API int deva_b200_readout_sparse_wide(const void* values, int64_t values_ld, int64_t values_rows,
                                                const int32_t* val_row, const int32_t* out_row, int n_groups,
                                                int rows_per_group, const int32_t* idx, const float* w, int ld_list,
                                                int top_k, int n_window, int q, void* workspace, float* out,
                                                int64_t ld_out, void* out_tok, deva_stream_t stream) {
  return readout_sparse(values, values_ld, values_rows, val_row, out_row, nullptr, n_groups, rows_per_group, idx, w,
                        ld_list, top_k, n_window, q, workspace, out, nullptr, 0, ld_out, out_tok, stream);
}

DEVA_B200_API int deva_b200_readout_sparse_scatter_wide(const void* values, int64_t values_ld, int64_t values_rows,
                                                        const int32_t* val_row, const int32_t* out_row,
                                                        const int32_t* owner, int n_groups, int rows_per_group,
                                                        const int32_t* idx, const float* w, int ld_list, int top_k,
                                                        int n_window, int q, void* workspace, float* const* rank_dst,
                                                        int n_ranks, int64_t ld_out, deva_stream_t stream) {
  return readout_sparse(values, values_ld, values_rows, val_row, out_row, owner, n_groups, rows_per_group, idx, w,
                        ld_list, top_k, n_window, q, workspace, nullptr, rank_dst, n_ranks, ld_out, nullptr, stream);
}

}  // extern "C"
