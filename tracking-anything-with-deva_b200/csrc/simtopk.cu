// Anisotropic-L2 similarity + per-query top-k + softmax, fused
// (reference: get_similarity + do_softmax, deva/model/memory_utils.py:6-76).
//
// sim[n,q] = s_n * ( sum_c mk_cn^2 * (-qe_cq) + sum_c mk_cn * (2 qk_cq qe_cq) - bsq_q ),  s_n = shrinkage_n / sqrt(CK)
// runs as ONE wgmma GEMM with K = 2*CK:   key row n = [ s*mk^2 | s*mk ],  query row q = [ -qe | 2*qk*qe ],
// and the  - s_n * bsq_q  term is applied in the epilogue.  fp32-equivalent accuracy comes from a
// three-term split of both operands into fp16 (hi, lo) pairs: D = Qh.Kh + Ql.Kh + Qh.Kl, fp32 accumulate
// (11+11 significand bits; the dropped Ql.Kl term is ~2^-22 relative).
//
// CTA = 64 queries x a contiguous range of 64-slot memory tiles; the query operand is TMA-loaded once and stays
// resident, key tiles stream through a 2-stage ring.  Two consumer warpgroups take alternating tiles: each runs the
// 64 x 64 wgmma of its tile, stages the accumulator in shared memory, and then two threads per query scan one half of
// the tile each with a running threshold (current k-th best), keeping their k best (value, slot) pairs in a
// bank-conflict-free shared-memory column: four candidate lists per query.  The memory axis can be split over several
// CTAs (grid.y); a small merge kernel picks the global top-k, applies the softmax, accumulates per-slot usage and
// scatters the dense fp16 affinity rows consumed by the readout GEMM.
#include <cuda_fp16.h>
#include <math_constants.h>

#include "common.h"
#include "ptx.cuh"
#include "tmap.h"

namespace b200 {
namespace simtopk {

constexpr int kMaxSplit = 4;        // max CTAs sharing one 64-query tile along the memory axis
constexpr int kMaxMergeLists = 16;  // candidate lists per query of one merge
constexpr int BQ = 64, BNK = 64, BK = 64;
constexpr int QTILE_BYTES = BQ * 128;   // 64 query rows x 64 halves
constexpr int KTILE_BYTES = BNK * 128;  // 64 key rows x 64 halves
constexpr int MAX_KB = 2;               // 2*CK/64 with CK <= 64
constexpr int KSTAGES = 2;
constexpr int GROUPS = 2;               // consumer warpgroups working on alternating tiles
constexpr int LISTS = 2 * GROUPS;       // candidate lists per query: (group, column half)
static_assert(kMaxSplit * LISTS <= kMaxMergeLists, "merge: candidate lists per query");
constexpr int THREADS = GROUPS * 128 + 32;  // warps 0..7 consumers, warp 8 TMA producer
constexpr int Q_BYTES = 2 * MAX_KB * QTILE_BYTES;  // hi/lo x k-blocks
constexpr int KSTAGE_BYTES = 2 * MAX_KB * KTILE_BYTES;
constexpr int LIST_BYTES = LISTS * 2 * kListCap * BQ * 4;
constexpr int STG_PITCH = BNK + 4;      // fp32 accumulator staging row pitch (conflict-free float4 row reads)
constexpr int STG_BYTES = GROUPS * BQ * STG_PITCH * 4;
constexpr int NS_BYTES = GROUPS * BNK * 4;
constexpr int THR_BYTES = LISTS * BQ * 4;  // each list publishes its running k-th best per query
constexpr int SMEM_BYTES = Q_BYTES + KSTAGES * KSTAGE_BYTES + LIST_BYTES + STG_BYTES + NS_BYTES + 256 + THR_BYTES;
static_assert(SMEM_BYTES <= 232448, "simtopk: shared-memory budget");

struct Params {
  int q, n_window, n_lead, kblocks, top_k;
  int tiles_total, tiles_per_split;
  int qpad;
  const float* neg_s;   // [n_window]  -shrinkage/sqrt(CK)
  const float* bsq;     // [q]
  float* part_val;      // [nsplit*LISTS][kListCap][qpad]
  int* part_idx;
  float* dense_out;     // DENSE mode: [q][ld_dense]
  long long ld_dense;
  const float* thr_floor;  // optional [q]: a lower bound of each query's k-th best similarity (temporal warm start)
};

// v[j] for a run-time j without spilling v to local memory: 5-level select tree (31 selects).
__device__ __forceinline__ float pick32(const float (&v)[32], int j) {
  float a[16], b[8], c[4], d[2];
#pragma unroll
  for (int i = 0; i < 16; ++i) a[i] = (j & 16) ? v[i + 16] : v[i];
#pragma unroll
  for (int i = 0; i < 8; ++i) b[i] = (j & 8) ? a[i + 8] : a[i];
#pragma unroll
  for (int i = 0; i < 4; ++i) c[i] = (j & 4) ? b[i + 4] : b[i];
#pragma unroll
  for (int i = 0; i < 2; ++i) d[i] = (j & 2) ? c[i + 2] : c[i];
  return (j & 1) ? d[1] : d[0];
}

// Per-thread running top-k: kListCap (32) candidate slots in a shared-memory column (entries >= top_k hold
// +inf), tracked as 4 groups of 8 with the group minima (value, slot, position) in registers.  Replacing the global
// minimum re-scans only its group: 16 shared loads + a handful of selects per insertion.
// Entries are ranked by (similarity descending, slot ascending): of two equal similarities the higher slot is the
// minimum and is evicted first.  A list scans its columns in ascending slot order and admits a column only above its
// k-th best, so it always holds exactly the top-k of the columns it has seen under that order, whatever the history
// of insertions (cold or warm-started).
struct TopK {
  float gmin[4];
  int gidx[4];
  int gpos[4];
  float thr;
  int minpos;
  // (v, n) ranks below (u, m)
  static __device__ __forceinline__ bool below(float v, int n, float u, int m) { return v < u || (v == u && n > m); }
  __device__ __forceinline__ void refresh() {
    float m01 = gmin[0]; int i01 = gidx[0], p01 = gpos[0];
    if (below(gmin[1], gidx[1], m01, i01)) { m01 = gmin[1]; i01 = gidx[1]; p01 = gpos[1]; }
    float m23 = gmin[2]; int i23 = gidx[2], p23 = gpos[2];
    if (below(gmin[3], gidx[3], m23, i23)) { m23 = gmin[3]; i23 = gidx[3]; p23 = gpos[3]; }
    const bool c = below(m23, i23, m01, i01);
    thr = c ? m23 : m01;
    minpos = c ? p23 : p01;
  }
  __device__ __forceinline__ void insert(float* lv, int* li, int row, float v, int n) {
    lv[minpos * BQ + row] = v;
    li[minpos * BQ + row] = n;
    const int g = minpos >> 3;
    const float* base = lv + (g * 8) * BQ + row;
    const int* ibase = li + (g * 8) * BQ + row;
    float x[8];
    int y[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { x[e] = base[e * BQ]; y[e] = ibase[e * BQ]; }
    float m = x[0]; int mi = y[0], mp = 0;
#pragma unroll
    for (int e = 1; e < 8; ++e)
      if (below(x[e], y[e], m, mi)) { m = x[e]; mi = y[e]; mp = e; }
    mp += g * 8;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (i == g) { gmin[i] = m; gidx[i] = mi; gpos[i] = mp; }
    refresh();
  }
};

template <bool DENSE>
__global__ void __launch_bounds__(THREADS, 1)
simtopk_kernel(const __grid_constant__ CUtensorMap map_qh, const __grid_constant__ CUtensorMap map_ql,
               const __grid_constant__ CUtensorMap map_kh, const __grid_constant__ CUtensorMap map_kl,
               const __grid_constant__ Params p) {
  // 1024-byte alignment (128B swizzle atoms) comes from the declaration: deriving an aligned pointer through an
  // integer cast would make the compiler lose the shared address space (generic LD/ST instead of LDS/STS).
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sQ = smem;                                   // [hi/lo][kb] query tiles, resident
  uint8_t* sK = smem + Q_BYTES;                         // [stage][hi/lo][kb] key tiles
  float* list_val = reinterpret_cast<float*>(sK + KSTAGES * KSTAGE_BYTES);   // [list][kListCap][BQ]
  int* list_idx = reinterpret_cast<int*>(list_val + LISTS * kListCap * BQ);
  float* stg = reinterpret_cast<float*>(list_idx + LISTS * kListCap * BQ);   // [group][BQ][STG_PITCH]
  float* ns = stg + GROUPS * BQ * STG_PITCH;                                 // [group][BNK]
  uint64_t* bars = reinterpret_cast<uint64_t*>(ns + GROUPS * BNK);
  uint64_t* q_full = bars;
  uint64_t* full = bars + 1;                    // [KSTAGES]
  uint64_t* empty = full + KSTAGES;             // [KSTAGES]
  volatile float* thr_pub = reinterpret_cast<volatile float*>(reinterpret_cast<uint8_t*>(bars) + 256);  // [LISTS][BQ]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * BQ;
  const int t_begin = blockIdx.y * p.tiles_per_split;
  const int t_end = min(p.tiles_total, t_begin + p.tiles_per_split);

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&map_qh); tma_prefetch_desc(&map_ql);
    tma_prefetch_desc(&map_kh); tma_prefetch_desc(&map_kl);
    mbar_init(q_full, 1);
    for (int i = 0; i < KSTAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 1); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(q_full, 2u * p.kblocks * QTILE_BYTES);
      for (int kb = 0; kb < p.kblocks; ++kb) {
        tma_load_2d(sQ + (0 * MAX_KB + kb) * QTILE_BYTES, &map_qh, q_full, kb * BK, q0);
        tma_load_2d(sQ + (1 * MAX_KB + kb) * QTILE_BYTES, &map_ql, q_full, kb * BK, q0);
      }
      int stage = 0;
      uint32_t phase = 0;
      for (int t = t_begin; t < t_end; ++t) {
        mbar_wait(&empty[stage], phase ^ 1);
        mbar_expect_tx(&full[stage], 2u * p.kblocks * KTILE_BYTES);
        uint8_t* dst = sK + stage * KSTAGE_BYTES;
        for (int kb = 0; kb < p.kblocks; ++kb) {
          tma_load_2d(dst + (0 * MAX_KB + kb) * KTILE_BYTES, &map_kh, &full[stage], kb * BK, t * BNK);
          tma_load_2d(dst + (1 * MAX_KB + kb) * KTILE_BYTES, &map_kl, &full[stage], kb * BK, t * BNK);
        }
        if (++stage == KSTAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  const int group = warp >> 2;        // 0: even local tiles, 1: odd local tiles
  const int tid = threadIdx.x & 127;  // thread within the group's warpgroup
  const int row = tid & (BQ - 1);     // query within the tile
  const int half = tid >> 6;          // 32-column half of the tile this thread scans
  const int list = group * 2 + half;
  const int qg = q0 + row;
  const float bsq = (qg < p.q) ? p.bsq[qg] : 0.f;
  const int top_k = p.top_k;
  // Nothing at or below a valid lower bound of the k-th best similarity can be in the top-k: with the bound taken from
  // the slots the previous frame selected, only a handful of candidates per query ever reach the insertion path.
  const float floor_thr = (!DENSE && p.thr_floor && qg < p.q) ? p.thr_floor[qg] : -CUDART_INF_F;
  float* lv = list_val + list * kListCap * BQ;
  int* li = list_idx + list * kListCap * BQ;
  float* my_stg = stg + group * BQ * STG_PITCH;
  float* my_ns = ns + group * BNK;
  TopK tk;
  if (!DENSE) {
    for (int j = 0; j < kListCap; ++j) {
      lv[j * BQ + row] = (j < top_k) ? -CUDART_INF_F : CUDART_INF_F;
      li[j * BQ + row] = -1;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      tk.gmin[i] = (i * 8 < top_k) ? -CUDART_INF_F : CUDART_INF_F;
      tk.gidx[i] = -1;
      tk.gpos[i] = i * 8;
    }
    tk.refresh();
    // The two halves scan disjoint columns of the SAME queries into separate lists.  Each publishes its running k-th
    // best; the other's value is a valid lower bound of the query's global k-th best (its list holds k real candidates
    // at least that large), so gating on it keeps every global top-k member while cutting the insertions of two
    // half-length lists to about those of one full-length list.  Stale reads are fine: the bound only grows.  A column
    // EQUAL to the other list's k-th best is still admitted: it may be a global top-k member that wins the tie by its
    // lower slot, and whether the other list has published that value yet depends on timing.
    thr_pub[list * BQ + row] = -CUDART_INF_F;
    named_bar_sync(3, GROUPS * 128);
  }
  volatile const float* thr_other = thr_pub + (list ^ 1) * BQ + row;
  mbar_wait(q_full, 0);
  const uint32_t q_base = smem_u32(sQ);
  for (int it = group; t_begin + it < t_end; it += GROUPS) {
    const int stage = it % KSTAGES;
    const int n0 = (t_begin + it) * BNK;
    float d[BNK / 2];
    mbar_wait(&full[stage], (it / KSTAGES) & 1);
    const uint32_t k_base = smem_u32(sK + stage * KSTAGE_BYTES);
    wgmma_fence();
    for (int kb = 0; kb < p.kblocks; ++kb) {
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t qh = wgmma_desc_sw128(q_base + (0 * MAX_KB + kb) * QTILE_BYTES + k * 32);
        const uint64_t ql = wgmma_desc_sw128(q_base + (1 * MAX_KB + kb) * QTILE_BYTES + k * 32);
        const uint64_t kh = wgmma_desc_sw128(k_base + (0 * MAX_KB + kb) * KTILE_BYTES + k * 32);
        const uint64_t kl = wgmma_desc_sw128(k_base + (1 * MAX_KB + kb) * KTILE_BYTES + k * 32);
        wgmma_f16<BNK>(d, ql, kh, (kb | k) != 0);
        wgmma_f16<BNK>(d, qh, kl, 1);
        wgmma_f16<BNK>(d, qh, kh, 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(d);
    if (tid == 0) mbar_arrive(&empty[stage]);
    named_bar_sync(1 + group, 128);  // the previous tile's staging / ns reads are done
    if (tid < BNK) {
      const int n = n0 + tid;
      my_ns[tid] = (n >= p.n_lead && n < p.n_window) ? p.neg_s[n] : -CUDART_INF_F;
    }
#pragma unroll
    for (int j = 0; j < BNK / 8; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = (warp & 3) * 16 + (lane >> 2) + 8 * i;
        *reinterpret_cast<float2*>(my_stg + r * STG_PITCH + 8 * j + 2 * (lane & 3)) =
            make_float2(d[4 * j + 2 * i], d[4 * j + 2 * i + 1]);
      }
    named_bar_sync(1 + group, 128);
    const float4* ns4 = reinterpret_cast<const float4*>(my_ns + half * 32);
    const float4* acc4 = reinterpret_cast<const float4*>(my_stg + row * STG_PITCH + half * 32);
    float v[32];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 s4 = ns4[j];
      const float4 a4 = acc4[j];
      v[4 * j + 0] = fmaf(s4.x, bsq, a4.x);
      v[4 * j + 1] = fmaf(s4.y, bsq, a4.y);
      v[4 * j + 2] = fmaf(s4.z, bsq, a4.z);
      v[4 * j + 3] = fmaf(s4.w, bsq, a4.w);
    }
    const int c0 = n0 + half * 32;
    if (DENSE) {
      if (qg < p.q) {
        float* dst = p.dense_out + (long long)qg * p.ld_dense + c0;
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (c0 + j < p.n_window) dst[j] = (v[j] == v[j]) ? v[j] : -CUDART_INF_F;
      }
    } else {
      // Bit j of `pending` = column j beats this query's current k-th best.  Lanes then retire their
      // pending candidates in lock-step (1st of every lane, 2nd of every lane, ...): the warp pays for
      // max-per-lane insertions per tile, not for every distinct column position.
      uint32_t pending = 0;
      const float gate = fmaxf(tk.thr, floor_thr);
      const float gate_other = *thr_other;
#pragma unroll
      for (int j = 0; j < 32; ++j) pending |= (v[j] > gate && v[j] >= gate_other) ? (1u << j) : 0u;
      while (__any_sync(0xffffffffu, pending != 0)) {
        if (pending) {
          const int j = __ffs(pending) - 1;
          pending &= pending - 1;
          const float x = pick32(v, j);
          if (x > tk.thr) tk.insert(lv, li, row, x, c0 + j);
        }
      }
      thr_pub[list * BQ + row] = tk.thr;
    }
  }
  if (!DENSE) {
    const long long base = ((long long)blockIdx.y * LISTS + list) * kListCap;
    for (int j = 0; j < top_k; ++j) {
      p.part_val[(base + j) * p.qpad + qg] = lv[j * BQ + row];
      p.part_idx[(base + j) * p.qpad + qg] = li[j * BQ + row];
    }
  }
}

// One warp per query: global top-k over the per-split candidate lists, softmax, usage, dense scatter.
constexpr int MERGE_WARPS = 8;
__global__ void __launch_bounds__(MERGE_WARPS * 32)
merge_kernel(const float* __restrict__ part_val, const int* __restrict__ part_idx, int nsplit, int top_k, int q,
             int qpad, int* __restrict__ out_idx, float* __restrict__ out_w, __half* __restrict__ P, long long ldP,
             float* __restrict__ use_cnt, int n_long, int add_long, int add_work, float* __restrict__ out_sim) {
  // row pitch = 4 mod 32: the staging writes of a warp (4 candidates x 8 queries) and the per-warp scans are conflict-free
  __shared__ float cv[MERGE_WARPS][kMaxMergeLists * kListCap + 4];
  __shared__ int ci[MERGE_WARPS][kMaxMergeLists * kListCap + 4];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qb = blockIdx.x * MERGE_WARPS;
  const int C = nsplit * top_k;
  // cooperative, sector-coalesced staging of the [C candidates] x [8 queries] tile (rows are qpad apart)
  for (int i = threadIdx.x; i < C * MERGE_WARPS; i += MERGE_WARPS * 32) {
    const int c = i / MERGE_WARPS, qo = i - c * MERGE_WARPS;
    const int s_ = c / top_k, j = c - s_ * top_k;
    const long long off = ((long long)s_ * kListCap + j) * qpad + qb + qo;
    const bool ok = qb + qo < q;
    cv[qo][c] = ok ? part_val[off] : -CUDART_INF_F;
    ci[qo][c] = ok ? part_idx[off] : -1;
  }
  __syncthreads();
  const int qi = qb + w;
  if (qi >= q) return;
  float sel_v = -CUDART_INF_F;
  int sel_i = 0;
  for (int round = 0; round < top_k; ++round) {
    float bv = -CUDART_INF_F;
    int bi = 0x7fffffff, bc = -1;
    for (int c = lane; c < C; c += 32) {
      const float x = cv[w][c];
      const int xi = ci[w][c];
      if (xi >= 0 && (x > bv || (x == bv && xi < bi))) { bv = x; bi = xi; bc = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      const int oc = __shfl_xor_sync(0xffffffffu, bc, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; bc = oc; }
    }
    if (bc >= 0 && (bc & 31) == lane) ci[w][bc] = -1;  // consumed
    if (lane == round) { sel_v = bv; sel_i = (bc >= 0) ? bi : 0; }
    __syncwarp();
  }
  const float vmax = __shfl_sync(0xffffffffu, sel_v, 0);
  float e = (lane < top_k && sel_v > -CUDART_INF_F) ? expf(sel_v - vmax) : 0.f;
  float sum = e;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float wgt = e / sum;
  out_idx[(long long)qi * kListCap + lane] = (lane < top_k) ? sel_i : 0;
  out_w[(long long)qi * kListCap + lane] = (lane < top_k) ? wgt : 0.f;
  if (out_sim) out_sim[(long long)qi * kListCap + lane] = (lane < top_k) ? sel_v : -CUDART_INF_F;
  if (lane < top_k) {
    if (P) P[(long long)qi * ldP + sel_i] = __float2half_rn(wgt);
    if (use_cnt && ((sel_i < n_long) ? add_long : add_work)) atomicAdd(use_cnt + sel_i, wgt);
  }
}

// Full softmax over the window for every query row (consolidation: memory_utils.py:66-71), plus the
// shrinkage read-out  sum_n p[n] * shr[n]  (memory_manager.py:273).  One block per query.
__global__ void __launch_bounds__(256)
row_softmax_kernel(const float* __restrict__ sim, long long ld_sim, int n_window, const float* __restrict__ shr,
                   __half* __restrict__ P, long long ldP, float* __restrict__ shr_out) {
  __shared__ float red[8];
  const int qi = blockIdx.x;
  const float* row = sim + (long long)qi * ld_sim;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float m = -CUDART_INF_F;
  for (int n = threadIdx.x; n < n_window; n += 256) m = fmaxf(m, row[n]);
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[w] = m;
  __syncthreads();
  m = red[0];
  for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int n = threadIdx.x; n < n_window; n += 256) s += expf(row[n] - m);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) red[w] = s;
  __syncthreads();
  s = 0.f;
  for (int i = 0; i < 8; ++i) s += red[i];
  __syncthreads();
  const float inv = 1.f / s;
  float acc = 0.f;
  for (int n = threadIdx.x; n < n_window; n += 256) {
    const float pn = expf(row[n] - m) * inv;
    P[(long long)qi * ldP + n] = __float2half_rn(pn);
    if (shr) acc += pn * shr[n];
  }
  if (shr_out) {
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) red[w] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int i = 0; i < 8; ++i) t += red[i];
      shr_out[qi] = t;
    }
  }
}

__global__ void tick_kernel(float* __restrict__ life, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) life[i] += 1.f;
}

// ======================================================================================================
// Wide selection (any top_k, in particular beyond the kListCap-entry running lists of simtopk_kernel).  One CTA per
// query selects exactly the top_k of its candidates under (similarity descending, slot ascending) by a radix select on
// the order-preserving uint32 image of the fp32 similarity: 8-bit digits from the top, each pass a shared-memory
// histogram of the candidates that still match the prefix, stopping as soon as the threshold digit's bin holds exactly
// the entries still needed.  If more candidates than needed share the threshold value, a second radix select over their
// slots (ascending) keeps the lowest ones.  A compaction pass then writes the selected entries in candidate order, and
// the softmax (max-subtracted, fp32), usage and affinity scatter follow over the top_k written entries.
// Candidates are either a dense similarity row (written by simtopk_kernel<true>; kept in shared memory when it fits,
// else re-read from global memory / L2 by every pass) or n candidate lists with explicit slot ids (the cross-rank merge).
// ======================================================================================================
constexpr int WIDE_THREADS = 512;
constexpr int WIDE_WARPS = WIDE_THREADS / 32;
constexpr int kWideRowCache = 24576;  // dense rows up to this many slots are kept in shared memory (96 KiB)
constexpr int kWideMergeCap = 16384;  // candidates per query of one list merge, kept in shared memory (128 KiB)
enum WideMode { WIDE_ROW_GLOBAL = 0, WIDE_ROW_SMEM = 1, WIDE_LISTS = 2 };

struct WideParams {
  const float* sim;        // rows: [q][ld_sim], slots [n_lead, n_window) are the candidates
  long long ld_sim;
  int n_lead, n_window;
  const float* part_val;   // lists: [n_cand][q_pitch] values and slot ids (id < 0 = empty)
  const int* part_idx;
  int n_cand, q_pitch;
  int q, top_k, ld_list;
  int* out_idx;            // [q][ld_list]
  float* out_w;
  float* out_sim;
  __half* P;               // optional [q][ldP]
  long long ldP;
  float* use_cnt;          // optional [n_window]
  int n_long, add_long, add_work;
};

// -0 is mapped to +0 first: the order compares values, so the two zeros tie and their slots decide, as in merge_kernel.
__device__ __forceinline__ uint32_t order_key(float v) {
  const uint32_t b = __float_as_uint(v == 0.f ? 0.f : v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Every lane of the warp calls this; lanes with `on` add one to hist[bin], one atomic per distinct bin of the warp.
__device__ __forceinline__ void hist_add(int* hist, uint32_t bin, bool on) {
  const unsigned act = __ballot_sync(0xffffffffu, on);
  if (on) {
    const unsigned peers = __match_any_sync(act, bin);
    if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[bin], __popc(peers));
  }
}

// Radix select of the k largest keys among the candidates i < n for which get(i, key) is true.  On return the selected
// set is { masked key > prefix } plus `k` (updated) of { masked key == prefix }; the result is true when that equal
// set holds exactly k candidates (all taken), false when it holds more (the keys are then fully resolved: mask = ~0).
template <class Get>
__device__ bool radix_select(Get get, int n, int& k, uint32_t& prefix, uint32_t& mask, int* hist, int* ctl) {
  const int lane = threadIdx.x & 31;
  prefix = 0;
  mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += WIDE_THREADS) hist[i] = 0;
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += WIDE_THREADS) {
      const int i = i0 + threadIdx.x;
      uint32_t key = 0;
      const bool on = i < n && get(i, key) && (key & mask) == prefix;
      hist_add(hist, (key >> shift) & 255u, on);
    }
    __syncthreads();
    if (threadIdx.x < 32) {  // bin holding the k-th largest: lane l scans bins 255-8l .. 248-8l
      int c[8], s = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { c[j] = hist[255 - (lane * 8 + j)]; s += c[j]; }
      int incl = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      int run = incl - s;
      if (run < k && k <= incl) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (run + c[j] >= k) { ctl[0] = 255 - (lane * 8 + j); ctl[1] = run; ctl[2] = c[j]; break; }
          run += c[j];
        }
      }
    }
    __syncthreads();
    const uint32_t bin = (uint32_t)ctl[0];
    const int above = ctl[1], cnt = ctl[2];
    __syncthreads();  // ctl is rewritten by the next pass
    prefix |= bin << shift;
    mask |= 0xffu << shift;
    k -= above;
    if (cnt == k) return true;
  }
  return false;
}

__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < WIDE_WARPS; ++w) t += red[w];
  __syncthreads();
  return t;
}

__device__ __forceinline__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = -CUDART_INF_F;
  for (int w = 0; w < WIDE_WARPS; ++w) t = fmaxf(t, red[w]);
  __syncthreads();
  return t;
}

template <int MODE>
__global__ void __launch_bounds__(WIDE_THREADS)
wide_select_kernel(const __grid_constant__ WideParams p) {
  extern __shared__ uint32_t wide_smem[];  // cached keys [n], then (lists) slot ids [n]
  __shared__ int hist[256];
  __shared__ int ctl[3];
  __shared__ int wcnt[WIDE_WARPS];
  __shared__ float red[WIDE_WARPS];
  const int qi = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = (MODE == WIDE_LISTS) ? p.n_cand : p.n_window - p.n_lead;
  const float* row = (MODE == WIDE_LISTS) ? nullptr : p.sim + (long long)qi * p.ld_sim + p.n_lead;
  uint32_t* skey = wide_smem;
  int* sid = reinterpret_cast<int*>(wide_smem + n);

  int n_active = n;
  if (MODE != WIDE_ROW_GLOBAL) {
    int cnt = 0;
    for (int i = threadIdx.x; i < n; i += WIDE_THREADS) {
      if (MODE == WIDE_LISTS) {
        const long long off = (long long)i * p.q_pitch + qi;
        const int id = p.part_idx[off];
        skey[i] = order_key(p.part_val[off]);
        sid[i] = id;
        cnt += id >= 0;
      } else {
        skey[i] = order_key(row[i]);
      }
    }
    if (MODE == WIDE_LISTS) n_active = (int)block_sum((float)cnt, red);  // exact: counts < 2^24
    __syncthreads();
  }
  // candidate i -> (key, slot id); false for an empty list entry
  auto fetch = [&](int i, uint32_t& key, int& id) -> bool {
    if (MODE == WIDE_ROW_GLOBAL) { key = order_key(row[i]); id = p.n_lead + i; return true; }
    key = skey[i];
    if (MODE == WIDE_ROW_SMEM) { id = p.n_lead + i; return true; }
    id = sid[i];
    return id >= 0;
  };
  const int k_sel = min(p.top_k, n_active);
  int k = k_sel;
  uint32_t prefix = 0, mask = 0, id_prefix = 0, id_mask = 0;
  bool exact = true;  // every candidate whose masked key equals the prefix is selected
  if (k > 0) {
    exact = radix_select([&](int i, uint32_t& key) { int id; return fetch(i, key, id); }, n, k, prefix, mask, hist, ctl);
    if (!exact) {  // more candidates share the threshold value than are needed: the lowest slots win
      const uint32_t thr = prefix;
      radix_select(
          [&](int i, uint32_t& key) {
            uint32_t v; int id;
            const bool on = fetch(i, v, id) && v == thr;
            key = ~(uint32_t)id;
            return on;
          },
          n, k, id_prefix, id_mask, hist, ctl);
    }
  }

  // compaction in candidate order: entry e of the output = the e-th selected candidate
  int* oi = p.out_idx + (long long)qi * p.ld_list;
  float* ow = p.out_w + (long long)qi * p.ld_list;
  float vmax = -CUDART_INF_F;
  int base = 0;
  for (int i0 = 0; i0 < n && base < k_sel; i0 += WIDE_THREADS) {
    const int i = i0 + threadIdx.x;
    uint32_t key = 0;
    int id = 0;
    bool sel = false;
    if (i < n && fetch(i, key, id)) {
      const uint32_t mk = key & mask;
      sel = mk > prefix || (mk == prefix && (exact || (~(uint32_t)id & id_mask) >= id_prefix));
    }
    const unsigned b = __ballot_sync(0xffffffffu, sel);
    if (lane == 0) wcnt[warp] = __popc(b);
    __syncthreads();
    int off = base, tot = 0;
    for (int w = 0; w < WIDE_WARPS; ++w) {
      off += (w < warp) ? wcnt[w] : 0;
      tot += wcnt[w];
    }
    off += __popc(b & ((1u << lane) - 1u));
    if (sel && off < k_sel) {
      const float v = key_value(key);
      oi[off] = id;
      ow[off] = v;  // raw similarity for now; the weight replaces it below
      vmax = fmaxf(vmax, v);
    }
    base += tot;
    __syncthreads();
  }
  vmax = block_max(vmax, red);  // also orders the entries written above before the reads below
  float s = 0.f;
  for (int e = threadIdx.x; e < k_sel; e += WIDE_THREADS) s += expf(ow[e] - vmax);
  s = block_sum(s, red);
  for (int e = threadIdx.x; e < p.ld_list; e += WIDE_THREADS) {
    if (e < k_sel) {
      const int id = oi[e];
      const float v = ow[e];
      const float w = expf(v - vmax) / s;
      ow[e] = w;
      if (p.out_sim) p.out_sim[(long long)qi * p.ld_list + e] = v;
      if (p.P) p.P[(long long)qi * p.ldP + id] = __float2half_rn(w);
      if (p.use_cnt && ((id < p.n_long) ? p.add_long : p.add_work)) atomicAdd(p.use_cnt + id, w);
    } else {
      oi[e] = 0;
      ow[e] = 0.f;
      if (p.out_sim) p.out_sim[(long long)qi * p.ld_list + e] = -CUDART_INF_F;
    }
  }
}

}  // namespace simtopk

namespace simtopk {
// Temporal warm start: thr[q] = min over the slots the PREVIOUS read selected for query q of their similarity to the
// CURRENT query, minus a margin.  The k-th best of the whole window is >= the k-th best of any k of its slots, so this is
// a valid lower bound; consecutive frames share most of their top-k, so it is tight.  One warp per query, one lane per
// slot; operands are the hi parts of the packed rows the GEMM uses, evaluated in fp32 with a rigorous allowance for the
// dropped low-order parts.  Any invalid slot -> -inf (no bound); so is a repeated slot, since the minimum over fewer
// than k distinct slots does not bound the k-th best.
__global__ void __launch_bounds__(256)
thr_floor_kernel(const int* __restrict__ prev_idx, int top_k, int q, int n_lead, int n_window, int kdim,
                 const __half* __restrict__ k_hi, const float* __restrict__ neg_s, const __half* __restrict__ q_hi,
                 const float* __restrict__ bsq, float* __restrict__ thr) {
  __shared__ float qrow[8][128];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qi = blockIdx.x * 8 + w;
  if (qi >= q) return;
  // hi parts only (half the L2 traffic): sum (qh+ql)(kh+kl) = sum qh.kh + R with |R| <= sum |qh.kh| * 2^-9.9 since
  // |ql| <= 2^-11 |qh| and |kl| <= 2^-11 |kh|; the bound is lowered by that much, which keeps it valid.
  for (int c = lane; c < kdim; c += 32) qrow[w][c] = __half2float(q_hi[(long long)qi * kdim + c]);
  __syncwarp();
  float sim = CUDART_INF_F;
  bool bad = false;
  const int n = (lane < top_k) ? prev_idx[(long long)qi * kListCap + lane] : -1;
  const unsigned in_list = (top_k >= 32) ? 0xffffffffu : (1u << top_k) - 1u;
  const unsigned same = __match_any_sync(0xffffffffu, n) & in_list;  // every lane takes part
  if (lane < top_k && __popc(same) > 1) bad = true;
  if (lane < top_k) {
    if (n < n_lead || n >= n_window) {
      bad = true;
    } else {
      const uint4* ph = reinterpret_cast<const uint4*>(k_hi + (long long)n * kdim);
      float acc = 0.f, mag = 0.f;
      for (int c8 = 0; c8 < kdim / 8; ++c8) {
        const uint4 vh = ph[c8];
        const __half2* h2 = reinterpret_cast<const __half2*>(&vh);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 a = __half22float2(h2[e]);
          const float t0 = a.x * qrow[w][c8 * 8 + 2 * e], t1 = a.y * qrow[w][c8 * 8 + 2 * e + 1];
          acc += t0 + t1;
          mag += fabsf(t0) + fabsf(t1);
        }
      }
      sim = fmaf(neg_s[n], bsq[qi], acc) - mag * (1.f / 512.f);
    }
  }
  bad = __any_sync(0xffffffffu, bad);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sim = fminf(sim, __shfl_xor_sync(0xffffffffu, sim, o));
  if (lane == 0) thr[qi] = (bad || !(sim == sim)) ? -CUDART_INF_F : sim - 1e-3f * (1.f + fabsf(sim));
}
}  // namespace simtopk

static int make_maps(CUtensorMap* m, const __half* q_hi, const __half* q_lo, int q, const __half* k_hi,
                     const __half* k_lo, int n_window, int ck) {
  const char* err = nullptr;
  const uint64_t kdim = 2ull * ck;
  if (make_tmap_2d(&m[0], TmapType::F16, q_hi, kdim, q, kdim * 2, 64, simtopk::BQ, &err) ||
      make_tmap_2d(&m[1], TmapType::F16, q_lo, kdim, q, kdim * 2, 64, simtopk::BQ, &err) ||
      make_tmap_2d(&m[2], TmapType::F16, k_hi, kdim, n_window, kdim * 2, 64, 64, &err) ||
      make_tmap_2d(&m[3], TmapType::F16, k_lo, kdim, n_window, kdim * 2, 64, 64, &err)) {
    set_error("simtopk: %s", err ? err : "tensor map");
    return 3;
  }
  return 0;
}


// Split of the memory axis over CTAs: minimise (waves) x (tiles per CTA), with a small per-split
// charge for the list warm-up every split repeats.
static int choose_split(int q_tiles, int tiles, int max_split) {
  const int sms = sm_count();
  int best = 1;
  long long best_cost = -1;
  for (int ns = 1; ns <= max_split && ns <= tiles; ++ns) {
    const long long waves = ceil_div((long long)q_tiles * ns, sms);
    const long long cost = waves * (ceil_div(tiles, ns) * 4 + 3);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = ns; }
  }
  return best;
}


// sim[q][ld_sim] (fp32, columns < n_window; slots < n_lead hold -inf) by the DENSE instantiation of simtopk_kernel: the
// similarity of deva_b200_sim_dense_softmax and of the wide top-k read.
static int dense_similarity(const __half* kh, const __half* kl, const float* neg_s, int n_window, int n_lead,
                            const __half* qh, const __half* ql, const float* bsq, int q, int ck, float* sim,
                            long long ld_sim, cudaStream_t s) {
  using namespace simtopk;
  CUtensorMap maps[4];
  if (int rc = make_maps(maps, qh, ql, q, kh, kl, n_window, ck)) return rc;
  Params p{};
  p.q = q; p.n_window = n_window; p.n_lead = n_lead; p.kblocks = 2 * ck / 64; p.top_k = 1;
  p.tiles_total = ceil_div(n_window, BNK);
  const int q_tiles = ceil_div(q, BQ);
  int nsplit = ceil_div(sm_count(), q_tiles);
  if (nsplit > p.tiles_total) nsplit = p.tiles_total;
  p.tiles_per_split = ceil_div(p.tiles_total, nsplit);
  nsplit = ceil_div(p.tiles_total, p.tiles_per_split);
  p.qpad = q_tiles * BQ;
  p.neg_s = neg_s; p.bsq = bsq;
  p.dense_out = sim; p.ld_dense = ld_sim;
  static bool configured_dev[kMaxDevices] = {false};  // function attributes are per device
  bool& configured = configured_dev[device_slot()];
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(simtopk_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    configured = true;
  }
  simtopk_kernel<true><<<dim3(q_tiles, nsplit), THREADS, SMEM_BYTES, s>>>(maps[0], maps[1], maps[2], maps[3], p);
  B200_LAUNCH_CHECK();
  return 0;
}

// One wide_select_kernel launch per query: rows cached in shared memory when they fit, candidate lists always.
static int wide_select(simtopk::WideParams& p, int n, cudaStream_t s) {
  using namespace simtopk;
  static bool configured_dev[kMaxDevices] = {false};  // function attributes are per device
  bool& configured = configured_dev[device_slot()];
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(wide_select_kernel<WIDE_ROW_SMEM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   kWideRowCache * 4));
    B200_CUDA(cudaFuncSetAttribute(wide_select_kernel<WIDE_LISTS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   kWideMergeCap * 8));
    configured = true;
  }
  if (p.sim == nullptr) {
    wide_select_kernel<WIDE_LISTS><<<p.q, WIDE_THREADS, (size_t)n * 8, s>>>(p);
  } else if (n <= kWideRowCache) {
    wide_select_kernel<WIDE_ROW_SMEM><<<p.q, WIDE_THREADS, (size_t)n * 4, s>>>(p);
  } else {
    wide_select_kernel<WIDE_ROW_GLOBAL><<<p.q, WIDE_THREADS, 0, s>>>(p);
  }
  B200_LAUNCH_CHECK();
  return 0;
}

static int tick_life(float* life_cnt, int n_lead, int n_long, int n_window, int count_long, int count_work,
                      cudaStream_t s) {
  // life += 1 for every slot whose usage is being counted (kv_memory_store.py:118-125)
  const int lo = count_long ? n_lead : n_long;
  const int hi = count_work ? n_window : n_long;
  if (hi > lo) {
    simtopk::tick_kernel<<<ceil_div(hi - lo, 256), 256, 0, s>>>(life_cnt + lo, hi - lo);
    B200_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" {

DEVA_B200_API size_t deva_b200_simtopk_workspace_bytes(int q) {
  const size_t qpad = (size_t)ceil_div(q, simtopk::BQ) * simtopk::BQ;
  return (size_t)simtopk::kMaxSplit * simtopk::LISTS * kListCap * qpad * 8;
}

// k_hi/k_lo [n_window, 2*ck] and q_hi/q_lo [q, 2*ck]: the packed rows written by deva_b200_pack_keys /
// deva_b200_pack_query.
DEVA_B200_API int deva_b200_sim_topk(const void* k_hi, const void* k_lo, const float* neg_s, int n_window, int n_lead,
                                     const void* q_hi, const void* q_lo, const float* bsq, int q, int ck, int top_k,
                                     void* workspace, int32_t* out_idx, float* out_w, void* affinity, int64_t ld_affinity,
                                     float* use_cnt, float* life_cnt, int n_long, int count_long, int count_work,
                                     float* out_sim, const int32_t* prev_idx, float* thr_ws, deva_stream_t stream) {
  using namespace simtopk;
  const __half *kh = H(k_hi), *kl = H(k_lo), *qh = H(q_hi), *ql = H(q_lo);
  __half* P = H(affinity);
  const cudaStream_t s = S(stream);
  B200_REQUIRE(ck == 32 || ck == 64, "simtopk: key_dim %d unsupported (32 or 64)", ck);
  B200_REQUIRE(top_k >= 1 && top_k <= kListCap, "simtopk: top_k %d out of range [1,%d]", top_k, kListCap);
  B200_REQUIRE(n_window - n_lead >= top_k, "simtopk: top_k %d exceeds the %d memory slots (the reference raises too)",
               top_k, n_window - n_lead);
  B200_REQUIRE(q >= 1 && n_lead >= 0 && n_lead < 8, "simtopk: bad q / n_lead");
  CUtensorMap maps[4];
  if (int rc = make_maps(maps, qh, ql, q, kh, kl, n_window, ck)) return rc;
  Params p{};
  p.q = q; p.n_window = n_window; p.n_lead = n_lead; p.kblocks = 2 * ck / 64; p.top_k = top_k;
  p.tiles_total = ceil_div(n_window, BNK);
  const int q_tiles = ceil_div(q, BQ);
  int nsplit = choose_split(q_tiles, p.tiles_total, kMaxSplit);
  p.tiles_per_split = ceil_div(p.tiles_total, nsplit);
  nsplit = ceil_div(p.tiles_total, p.tiles_per_split);
  p.qpad = q_tiles * BQ;
  p.neg_s = neg_s; p.bsq = bsq;
  p.part_val = reinterpret_cast<float*>(workspace);
  p.part_idx = reinterpret_cast<int*>(p.part_val + (size_t)kMaxSplit * LISTS * kListCap * p.qpad);
  static bool configured_dev[kMaxDevices] = {false};  // function attributes are per device
  bool& configured = configured_dev[device_slot()];
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(simtopk_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    B200_CUDA(cudaFuncSetAttribute(simtopk_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    configured = true;
  }
  if (P) B200_CUDA(cudaMemsetAsync(P, 0, (size_t)q * ld_affinity * sizeof(__half), s));
  if (prev_idx) {
    B200_REQUIRE(thr_ws != nullptr, "simtopk: prev_idx needs the thr_ws scratch ([q] floats)");
    thr_floor_kernel<<<ceil_div(q, 8), 256, 0, s>>>(prev_idx, top_k, q, n_lead, n_window, 2 * ck, kh, neg_s, qh, bsq,
                                                    thr_ws);
    B200_LAUNCH_CHECK();
    p.thr_floor = thr_ws;
  }
  simtopk_kernel<false><<<dim3(q_tiles, nsplit), THREADS, SMEM_BYTES, s>>>(maps[0], maps[1], maps[2], maps[3], p);
  B200_LAUNCH_CHECK();
  merge_kernel<<<ceil_div(q, MERGE_WARPS), MERGE_WARPS * 32, 0, s>>>(
      p.part_val, p.part_idx, nsplit * LISTS, top_k, q, p.qpad, out_idx, out_w, P, ld_affinity, use_cnt, n_long, count_long,
      count_work, out_sim);
  B200_LAUNCH_CHECK();
  if (life_cnt) {
    if (int rc = tick_life(life_cnt, n_lead, n_long, n_window, count_long, count_work, s)) return rc;
  }
  return 0;
}

// Global top-k + softmax over `n_lists` candidate lists per query (layout [n_lists][kListCap][qpad], entries with
// idx < 0 are empty): the cross-rank merge of a bank-sharded read, and the second stage of deva_b200_sim_topk.
DEVA_B200_API int deva_b200_merge_lists(const float* part_val, const int32_t* part_idx, int n_lists, int top_k, int q,
                                        int q_pitch, int32_t* out_idx, float* out_w, float* out_sim,
                                        deva_stream_t stream) {
  using namespace simtopk;
  const cudaStream_t s = S(stream);
  B200_REQUIRE(n_lists >= 1 && n_lists <= kMaxMergeLists, "merge: n_lists %d out of range [1,%d]", n_lists, kMaxMergeLists);
  B200_REQUIRE(top_k >= 1 && top_k <= kListCap && q >= 1 && q_pitch >= q, "merge: bad shape");
  merge_kernel<<<ceil_div(q, MERGE_WARPS), MERGE_WARPS * 32, 0, s>>>(part_val, part_idx, n_lists, top_k, q, q_pitch,
                                                                    out_idx, out_w, nullptr, 0, nullptr, 0, 0, 0, out_sim);
  B200_LAUNCH_CHECK();
  return 0;
}

DEVA_B200_API int deva_b200_sim_dense_softmax(const void* k_hi, const void* k_lo, const float* neg_s,
                                              const float* shrinkage, int n_window, int n_lead, const void* q_hi,
                                              const void* q_lo, const float* bsq, int q, int ck, float* sim_ws,
                                              int64_t ld_sim, void* affinity, int64_t ld_affinity, float* shr_out,
                                              deva_stream_t stream) {
  using namespace simtopk;
  const __half *kh = H(k_hi), *kl = H(k_lo), *qh = H(q_hi), *ql = H(q_lo);
  __half* P = H(affinity);
  const cudaStream_t s = S(stream);
  B200_REQUIRE(ck == 32 || ck == 64, "simdense: key_dim %d unsupported (32 or 64)", ck);
  B200_REQUIRE(q >= 1 && n_window > n_lead && n_lead >= 0 && n_lead < 8, "simdense: bad shape");
  if (int rc = dense_similarity(kh, kl, neg_s, n_window, n_lead, qh, ql, bsq, q, ck, sim_ws, ld_sim, s)) return rc;
  row_softmax_kernel<<<q, 256, 0, s>>>(sim_ws, ld_sim, n_window, shrinkage, P, ld_affinity, shr_out);
  B200_LAUNCH_CHECK();
  return 0;
}


// ---- wide top-k read (any top_k; the path for top_k > kListCap) ----
static long long wide_ld_sim(int n_window) { return ((long long)n_window + 31) / 32 * 32; }

DEVA_B200_API size_t deva_b200_sim_topk_wide_workspace_bytes(int q, int n_window) {
  if (q < 1 || n_window < 1) return 0;
  return (size_t)q * (size_t)wide_ld_sim(n_window) * sizeof(float);
}

DEVA_B200_API int deva_b200_sim_topk_wide(const void* k_hi, const void* k_lo, const float* neg_s, int n_window,
                                          int n_lead, const void* q_hi, const void* q_lo, const float* bsq, int q, int ck,
                                          int top_k, void* workspace, int32_t* out_idx, float* out_w, int ld_list,
                                          void* affinity, int64_t ld_affinity, float* use_cnt, float* life_cnt,
                                          int n_long, int count_long, int count_work, float* out_sim,
                                          deva_stream_t stream) {
  using namespace simtopk;
  const cudaStream_t s = S(stream);
  B200_REQUIRE(ck == 32 || ck == 64, "simtopk_wide: key_dim %d unsupported (32 or 64)", ck);
  B200_REQUIRE(top_k >= 1, "simtopk_wide: top_k %d must be at least 1", top_k);
  B200_REQUIRE(n_window - n_lead >= top_k,
               "simtopk_wide: top_k %d exceeds the %d memory slots (the reference raises too)", top_k, n_window - n_lead);
  B200_REQUIRE(q >= 1 && n_lead >= 0 && n_lead < 8, "simtopk_wide: bad q / n_lead");
  B200_REQUIRE(ld_list >= top_k && ld_list % 32 == 0, "simtopk_wide: ld_list %d must be a multiple of 32 and >= top_k %d",
               ld_list, top_k);
  B200_REQUIRE(workspace != nullptr && out_idx != nullptr && out_w != nullptr, "simtopk_wide: missing buffer");
  float* sim = reinterpret_cast<float*>(workspace);
  const long long ld_sim = wide_ld_sim(n_window);
  if (int rc = dense_similarity(H(k_hi), H(k_lo), neg_s, n_window, n_lead, H(q_hi), H(q_lo), bsq, q, ck, sim, ld_sim, s))
    return rc;
  __half* P = H(affinity);
  if (P) B200_CUDA(cudaMemsetAsync(P, 0, (size_t)q * ld_affinity * sizeof(__half), s));
  WideParams p{};
  p.sim = sim; p.ld_sim = ld_sim; p.n_lead = n_lead; p.n_window = n_window;
  p.q = q; p.top_k = top_k; p.ld_list = ld_list;
  p.out_idx = out_idx; p.out_w = out_w; p.out_sim = out_sim;
  p.P = P; p.ldP = ld_affinity;
  p.use_cnt = use_cnt; p.n_long = n_long; p.add_long = count_long; p.add_work = count_work;
  if (int rc = wide_select(p, n_window - n_lead, s)) return rc;
  if (life_cnt) {
    if (int rc = tick_life(life_cnt, n_lead, n_long, n_window, count_long, count_work, s)) return rc;
  }
  return 0;
}

DEVA_B200_API int deva_b200_merge_lists_wide(const float* part_val, const int32_t* part_idx, int n_lists, int ld_list,
                                             int top_k, int q, int q_pitch, int32_t* out_idx, float* out_w,
                                             float* out_sim, deva_stream_t stream) {
  using namespace simtopk;
  B200_REQUIRE(n_lists >= 1 && n_lists <= kMaxMergeLists, "merge_wide: n_lists %d out of range [1,%d]", n_lists,
               kMaxMergeLists);
  B200_REQUIRE(top_k >= 1 && ld_list >= top_k && ld_list % 32 == 0,
               "merge_wide: top_k %d must be in [1, ld_list] and ld_list %d a multiple of 32", top_k, ld_list);
  B200_REQUIRE((long long)n_lists * ld_list <= kWideMergeCap, "merge_wide: %d lists of %d entries exceed %d candidates",
               n_lists, ld_list, kWideMergeCap);
  B200_REQUIRE(q >= 1 && q_pitch >= q, "merge_wide: bad shape");
  WideParams p{};
  p.part_val = part_val; p.part_idx = part_idx; p.n_cand = n_lists * ld_list; p.q_pitch = q_pitch;
  p.q = q; p.top_k = top_k; p.ld_list = ld_list;
  p.out_idx = out_idx; p.out_w = out_w; p.out_sim = out_sim;
  return wide_select(p, p.n_cand, S(stream));
}

}  // extern "C"
