#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stddef.h>

namespace b200 {
constexpr int kListCap = 32;  // max top_k; also the row pitch of the idx / weight outputs
constexpr int kMaxSplit = 4;  // max CTAs sharing one 64-query tile along the memory axis

size_t simtopk_workspace_bytes(int q);

// Top-k + softmax read.  All slot indices are relative to the window start.
//   k_hi/k_lo [n_window, 2*ck] fp16 packed key rows, neg_s [n_window]; slots < n_lead are masked.
//   q_hi/q_lo [q, 2*ck] fp16 packed query rows, bsq [q].
//   out_idx/out_w [q, kListCap] sorted by descending similarity (entries >= top_k are zero).
//   P (optional) [q, ldP] fp16 dense affinity rows, zero-filled then scattered.
//   use_cnt/life_cnt (optional) [n_window]; slots < n_long are the long-term region.
int launch_sim_topk(const __half* k_hi, const __half* k_lo, const float* neg_s, int n_window, int n_lead,
                    const __half* q_hi, const __half* q_lo, const float* bsq, int q, int ck, int top_k,
                    void* workspace, int* out_idx, float* out_w, __half* P, long long ldP, float* use_cnt,
                    float* life_cnt, int n_long, int count_long, int count_work, float* out_sim, const int* prev_idx,
                    float* thr_ws, cudaStream_t stream);
// out_sim (optional): [q, kListCap] raw similarities of the selected slots (descending), -inf beyond top_k
// prev_idx (optional, with thr_ws [q]): the out_idx of the previous read of the SAME window (slot numbering unchanged;
//   may alias out_idx): those slots' similarities to the current queries bound each query's k-th best from below, and
//   the streaming top-k only inserts candidates above that bound (exact; see thr_floor_kernel).

constexpr int kMaxMergeLists = 16;
int launch_merge_lists(const float* part_val, const int* part_idx, int n_lists, int top_k, int q, int qpad, int* out_idx,
                       float* out_w, float* out_sim, cudaStream_t stream);

// Full-softmax variant (consolidation): sim_ws [q, ld_sim] fp32 scratch, P [q, ldP] fp16,
// shr_out[q] = sum_n P[q,n] * shr[n] (optional).
int launch_sim_dense_softmax(const __half* k_hi, const __half* k_lo, const float* neg_s, const float* shr,
                             int n_window, int n_lead, const __half* q_hi, const __half* q_lo, const float* bsq,
                             int q, int ck, float* sim_ws, long long ld_sim, __half* P, long long ldP, float* shr_out,
                             cudaStream_t stream);
}  // namespace b200
