/*
 * deva_b200 - C ABI of the H100-native temporal-propagation kernels behind DEVA's
 * DEVAInferenceCore.step / MemoryManager API.
 *
 * The reference (hkchengrex/Tracking-Anything-with-DEVA @ 404a112) is pure Python/PyTorch and has no
 * FFI of its own; the boundary it exposes for this path is the set of Python call sites cited on each
 * entry point below.  A maintainer binds this library with ctypes (see INTEGRATION.md); the shipped
 * drop-in package does exactly that (tracking-anything-with-deva_b200/deva/_native.py).
 *
 * Conventions
 *  - every pointer is a CUDA device pointer unless marked HOST; fp16 buffers are passed as void*;
 *  - `stream` is a cudaStream_t (0 = legacy default stream); calls only enqueue work and never
 *    synchronise; inputs are borrowed until the enqueued work completes, outputs are caller-allocated;
 *  - return 0 on success; otherwise a non-zero code, with text available from deva_b200_last_error()
 *    (thread-local).  The Python side raises RuntimeError, mirroring the reference's exceptions;
 *  - "window" = the contiguous run of valid memory slots of one bucket's bank; slot indices in the
 *    outputs are relative to the window start.  The first `n_lead` (< 8) slots of a window are
 *    alignment padding and are masked out.
 */
#ifndef DEVA_B200_H_
#define DEVA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* v29: deva_b200_sam_mask_stats, deva_b200_sam_mask_compact, deva_b200_sam_nms(_workspace_bytes) and
 * deva_b200_sam_mask_write (Segment Anything's automatic masks from the low-resolution logits).
 * v28: deva_b200_sim_topk_wide(_workspace_bytes), deva_b200_merge_lists_wide, deva_b200_readout_sparse_wide(_workspace_bytes)
 * and deva_b200_readout_sparse_scatter_wide (memory reads at any top_k, top-k lists at a caller-given pitch ld_list).
 * v27: deva_b200_conv2d takes flat spatial tiles, th = 0 and tw = 128 (stride 1, no out_pool4): 128 consecutive output
 * pixels of one image in row-major order.
 * v26: deva_b200_pil_resample_u8 and deva_b200_mask_nearest_ids (the dataset readers' soft masks and detection masks
 * resized on the device).
 * v25: deva_b200_jpeg_decode_workspace_bytes and deva_b200_jpeg_decode (baseline JPEG files decoded on the device).
 * v24: deva_b200_png_decode_workspace_bytes and deva_b200_png_decode (the post-processing passes' PNGs decoded on the
 * device).
 * v23: deva_b200_rle_bound, deva_b200_rle_workspace_bytes and deva_b200_rle_encode (BURST's per-segment COCO RLE encoded
 * on the device).
 * v22: deva_b200_jpeg_bound, deva_b200_jpeg_workspace_bytes and deva_b200_jpeg_encode (result JPEGs encoded on the
 * device).
 * v21: deva_b200_png_bound, deva_b200_png_workspace_bytes and deva_b200_png_encode (result PNGs encoded on the device).
 * v20: dropped deva_b200_up2_add and deva_b200_cbam (single-fp16 residual stream); deva_b200_up2_add_split requires skip_lo
 * and raw / raw_lo.
 * v19: deva_b200_mask_stats(_workspace_bytes), deva_b200_mask_scored_argmax and deva_b200_mask_last_cover (detector
 * masks -> detection id map).
 * v18: dropped conv split_mode 1, the split twins' relu_lo and hi-only pooling, gru, nhwc_to_nchw, enable_peer_access.
 * v16: deva_b200_label_areas and deva_b200_label_to_index (unsupervised DAVIS 2017 object limit).
 * v15: deva_b200_pano_joint_hist and deva_b200_pano_remap (video panoptic metrics and stuff merging).
 * v14: deva_b200_prob_to_scores and deva_b200_scores_to_ids (multi-scale / flip score export and merge).
 * v13: deva_b200_prob_to_segments (the result savers' id map, id image, overlay, areas and boxes in one pass).
 * v12: deva_b200_ingest_rgb8_resize and deva_b200_mask_nearest (frame and first-frame mask resized on the device).
 * v11: deva_b200_cbam / deva_b200_cbam_split take a larger scratch buffer (64 pooling slices) and require c = 8 x a divisor
 * of 256; deva_b200_conv2d requires cout_pad <= 2048 (<= 1024 with a rank-1 input): the layer's bias lives in shared memory. */
#define DEVA_B200_ABI_VERSION 29
#define DEVA_B200_LIST_PITCH 32 /* row pitch of deva_b200_sim_topk's outputs == its max top_k (wider: the _wide calls) */
#define DEVA_B200_MAX_GROUPS 256 /* objects per deva_b200_readout call */
#define DEVA_B200_MAX_SEGMENT_CHANNELS 8192 /* channels per deva_b200_prob_to_segments call */
#define DEVA_B200_MASK_SMEM_COUNTERS 8192 /* per-mask counters of one mask call kept in shared memory, else global */

typedef void* deva_stream_t; /* cudaStream_t */

#if defined(__GNUC__)
#define DEVA_B200_API __attribute__((visibility("default")))
#else
#define DEVA_B200_API
#endif

DEVA_B200_API int deva_b200_abi_version(void);
DEVA_B200_API const char* deva_b200_last_error(void);
/* Number of kernels this library has launched in the calling process (bench.py reports it). */
DEVA_B200_API uint64_t deva_b200_launch_count(void);
/* 0 when the current CUDA device can run the sm_90a kernels. */
DEVA_B200_API int deva_b200_device_check(void);

/* ---- query side ------------------------------------------------------------------------------------
 * Packs the per-frame query operand of get_similarity (deva/model/memory_utils.py:24-32):
 * row q = [ -qe[:,q] | 2*qk[:,q]*qe[:,q] ] split into fp16 (hi, lo), and bsq[q] = sum_c qe*qk^2.
 * Element (c, q) of qk/qe is read at c*stride_c + q*stride_q (channel-major [CK,Q]: stride_c=Q, stride_q=1).
 * q_hi/q_lo: [q, 2*ck] fp16;  bsq: [q] fp32.  ck in {32, 64}. */
DEVA_B200_API int deva_b200_pack_query(const float* qk, const float* qe, int64_t stride_c, int64_t stride_q, int ck, int q,
                         void* q_hi, void* q_lo, float* bsq, deva_stream_t stream);

/* ---- bank append -----------------------------------------------------------------------------------
 * Replaces the torch.cat growth of KeyValueMemoryStore.add (deva/inference/kv_memory_store.py:97-116):
 * writes `n` new tokens at the destination pointers (already offset to the first new slot).
 * key/selection element (c, t) at c*stride_c + t*stride_t; shrinkage [n].  selection/raw_sel may be NULL.
 * k_hi/k_lo: [n, 2*ck] fp16 rows [ s*k^2 | s*k ], s = shrinkage/sqrt(ck);  neg_s: [n] = -s;
 * raw_key/raw_sel: [n, ck] fp32 token-major copies;  raw_shr: [n]. */
DEVA_B200_API int deva_b200_pack_keys(const float* key, const float* selection, int64_t stride_c, int64_t stride_t,
                        const float* shrinkage, int ck, int n, void* k_hi, void* k_lo, float* neg_s, float* raw_key,
                        float* raw_sel, float* raw_shr, deva_stream_t stream);
/* Value rows fp32 src[r, j] (ld_src) -> fp16 dst[r, j] (ld_dst), r < rows, j < n
 * (MemoryManager.add_memory, deva/inference/memory_manager.py:199-205). */
DEVA_B200_API int deva_b200_append_values(const float* src, int64_t ld_src, void* dst, int64_t ld_dst, int rows, int n,
                            deva_stream_t stream);

/* ---- memory read -----------------------------------------------------------------------------------
 * get_similarity + do_softmax(top_k, inplace, return_usage) (deva/model/memory_utils.py:6-76) and the
 * usage bookkeeping of MemoryManager.match_memory / update_bucket_usage
 * (deva/inference/memory_manager.py:115-150, kv_memory_store.py:118-125), fused.
 *   workspace: deva_b200_simtopk_workspace_bytes(q) bytes of scratch;
 *   out_idx/out_w: [q, 32] int32 / fp32, entries sorted by descending similarity, zero beyond top_k;
 *   affinity (optional): [q, ld_affinity] fp16 dense rows (zero-filled, top_k non-zeros per row) for
 *                        deva_b200_readout;
 *   use_cnt/life_cnt (optional): [n_window] fp32 counters; slots < n_long are long-term memory;
 *   count_long/count_work: which region(s) receive usage (+= affinity row sums) and life (+= 1).
 * Ties: the selection is the top_k of the window's slots [n_lead, n_window) under the order (similarity descending,
 * slot ascending), where the similarity is the kernel's fp32 value; of bit-identical keys the lower slots are kept.
 * The result is deterministic and the same with or without prev_idx. */
DEVA_B200_API size_t deva_b200_simtopk_workspace_bytes(int q);
DEVA_B200_API int deva_b200_sim_topk(const void* k_hi, const void* k_lo, const float* neg_s, int n_window, int n_lead,
                       const void* q_hi, const void* q_lo, const float* bsq, int q, int ck, int top_k,
                       void* workspace, int32_t* out_idx, float* out_w, void* affinity, int64_t ld_affinity,
                       float* use_cnt, float* life_cnt, int n_long, int count_long, int count_work, float* out_sim,
                       const int32_t* prev_idx, float* thr_ws, deva_stream_t stream);
/* prev_idx (optional, with thr_ws: [q] fp32 scratch): out_idx of the PREVIOUS read of the same window (same slot numbering;
 * may alias out_idx).  Temporal warm start: the similarities of those top_k slots to the current queries bound every
 * query's k-th best from below, so the streaming top-k inserts only the few candidates above that bound - the result
 * is unchanged (exact), the epilogue work drops several-fold.  Pass NULL after any compaction / re-numbering.  A row
 * whose first top_k entries hold a slot outside [n_lead, n_window) or repeat a slot gives that query no bound (it is
 * read cold), since fewer than top_k distinct slots bound nothing. */
/* out_sim (optional): fp32 [q, 32] raw similarities of the selected slots (descending; -inf beyond top_k) - what a
 * bank-sharded read exchanges between ranks.
 *
 * deva_b200_merge_lists: global top-k + softmax over n_lists (<= 16) candidate lists per query, layout
 * part_val/part_idx [n_lists][32][q_pitch] (query index fastest; idx < 0 = empty entry).  It is the cross-rank merge of a
 * memory bank sharded along the slot axis (SURVEY section 8e): every rank all-gathers the (similarity, global slot) lists
 * of all ranks and obtains the identical global top-k set and softmax weights. */
DEVA_B200_API int deva_b200_merge_lists(const float* part_val, const int32_t* part_idx, int n_lists, int top_k, int q,
                                        int q_pitch, int32_t* out_idx, float* out_w, float* out_sim,
                                        deva_stream_t stream);
/* get_similarity + do_softmax without top-k (max-subtracted branch, memory_utils.py:66-71) as used by
 * MemoryManager.consolidation (memory_manager.py:262-273).  sim_ws: [q, ld_sim] fp32 scratch;
 * affinity: [q, ld_affinity] fp16;  shr_out[q] = sum_n affinity[q,n]*shrinkage[n] (optional). */
/* ---- wide read: the same read at any top_k (1 <= top_k <= n_window - n_lead), lists at pitch ld_list --------------
 * deva_b200_sim_topk_wide: the similarity of deva_b200_sim_dense_softmax (same kernel, same fp32 values) written to
 * workspace (deva_b200_sim_topk_wide_workspace_bytes(q, n_window) bytes: q rows of n_window rounded up to 32 floats),
 * then per query an exact radix select of the top_k slots of [n_lead, n_window) under (similarity descending, slot
 * ascending) - the tie rule of deva_b200_sim_topk, so for top_k <= 32 both select the same set - and the softmax
 * (max-subtracted, fp32) over them.
 *   out_idx/out_w (and out_sim, optional): [q, ld_list] int32 / fp32, ld_list a multiple of 32 and >= top_k; entries
 *     0 .. top_k-1 hold the selected slots in ASCENDING SLOT order (not by similarity), entries beyond are slot 0,
 *     weight 0, similarity -inf;
 *   affinity, use_cnt, life_cnt, n_long, count_long, count_work: as deva_b200_sim_topk.  There is no warm start.
 * A row of up to 24576 candidates is kept in shared memory during the select; a longer one is re-read from global
 * memory by every radix pass.  Errors: top_k < 1, top_k > n_window - n_lead, a bad ld_list.
 *
 * deva_b200_merge_lists_wide: deva_b200_merge_lists at any top_k: part_val/part_idx [n_lists][ld_list][q_pitch]
 * (n_lists <= 16, n_lists * ld_list <= 16384, idx < 0 = empty entry; the slot ids of one query must be distinct);
 * outputs [q, ld_list] as above, the selected candidates in input order (list by list, entry by entry), the same
 * order on every rank that passes the same lists.  If a query has fewer than top_k non-empty candidates, all of them
 * are taken and the remaining entries are empty. */
DEVA_B200_API size_t deva_b200_sim_topk_wide_workspace_bytes(int q, int n_window);
DEVA_B200_API int deva_b200_sim_topk_wide(const void* k_hi, const void* k_lo, const float* neg_s, int n_window,
                                          int n_lead, const void* q_hi, const void* q_lo, const float* bsq, int q, int ck,
                                          int top_k, void* workspace, int32_t* out_idx, float* out_w, int ld_list,
                                          void* affinity, int64_t ld_affinity, float* use_cnt, float* life_cnt,
                                          int n_long, int count_long, int count_work, float* out_sim,
                                          deva_stream_t stream);
DEVA_B200_API int deva_b200_merge_lists_wide(const float* part_val, const int32_t* part_idx, int n_lists, int ld_list,
                                             int top_k, int q, int q_pitch, int32_t* out_idx, float* out_w,
                                             float* out_sim, deva_stream_t stream);
DEVA_B200_API int deva_b200_sim_dense_softmax(const void* k_hi, const void* k_lo, const float* neg_s, const float* shrinkage,
                                int n_window, int n_lead, const void* q_hi, const void* q_lo, const float* bsq,
                                int q, int ck, float* sim_ws, int64_t ld_sim, void* affinity, int64_t ld_affinity,
                                float* shr_out, deva_stream_t stream);
/* MemoryManager._readout (deva/inference/memory_manager.py:64-75):
 * out[out_row[g] + r, j] = sum_n values[val_row[g] + r, n] * affinity[j, n]
 * for g < n_groups, r < rows_per_group (multiple of 128), j < q, n < n_window.
 * values: fp16 [values_rows, values_ld] already offset to the window start; val_row/out_row: HOST int32 arrays. */
DEVA_B200_API int deva_b200_readout(const void* values, int64_t values_ld, int64_t values_rows, const int32_t* val_row,
                      const int32_t* out_row, int n_groups, int rows_per_group, const void* affinity,
                      int64_t ld_affinity, int n_window, int q, float* out, int64_t ld_out, void* out_tok, deva_stream_t stream);
/* out_tok (optional; when non-NULL it replaces `out`): fp16 token-major result
 * out_tok[(object*q + j)*rows_per_group + r] with object = out_row[g] / rows_per_group - the layout the NHWC
 * decoder kernels consume. */

/* Same read-out with the affinity operand generated on chip: instead of a dense [q, n_window] fp16 matrix the
 * kernel takes the top-k lists written by deva_b200_sim_topk (idx/w: [q, 32]) and builds each 256-query x 64-slot
 * affinity tile in shared memory (zeroed stage buffers + scatter of the ~top_k*256*64/n_window non-zeros), so the
 * dense affinity never exists in HBM and only the value operand streams through TMA.
 * workspace: deva_b200_readout_sparse_workspace_bytes(q, n_window) bytes (per-tile bucket offsets + entries). */
DEVA_B200_API size_t deva_b200_readout_sparse_workspace_bytes(int q, int n_window);
DEVA_B200_API int deva_b200_readout_sparse(const void* values, int64_t values_ld, int64_t values_rows,
                                           const int32_t* val_row, const int32_t* out_row, int n_groups,
                                           int rows_per_group, const int32_t* idx, const float* w, int top_k,
                                           int n_window, int q, void* workspace, float* out, int64_t ld_out,
                                           void* out_tok, deva_stream_t stream);
/* The sparse read-outs with lists at pitch ld_list (a multiple of 32, top_k <= ld_list): the lists of
 * deva_b200_sim_topk_wide / deva_b200_merge_lists_wide.  workspace: deva_b200_readout_sparse_wide_workspace_bytes(q,
 * n_window, ld_list) bytes.  With ld_list = 32 they equal deva_b200_readout_sparse(_scatter). */
DEVA_B200_API size_t deva_b200_readout_sparse_wide_workspace_bytes(int q, int n_window, int ld_list);
DEVA_B200_API int deva_b200_readout_sparse_wide(const void* values, int64_t values_ld, int64_t values_rows,
                                                const int32_t* val_row, const int32_t* out_row, int n_groups,
                                                int rows_per_group, const int32_t* idx, const float* w, int ld_list,
                                                int top_k, int n_window, int q, void* workspace, float* out,
                                                int64_t ld_out, void* out_tok, deva_stream_t stream);
DEVA_B200_API int deva_b200_readout_sparse_scatter_wide(const void* values, int64_t values_ld, int64_t values_rows,
                                                        const int32_t* val_row, const int32_t* out_row,
                                                        const int32_t* owner, int n_groups, int rows_per_group,
                                                        const int32_t* idx, const float* w, int ld_list, int top_k,
                                                        int n_window, int q, void* workspace, float* const* rank_dst,
                                                        int n_ranks, int64_t ld_out, deva_stream_t stream);
/* Bank-sharded read (one video, slots split over the ranks of an NVLink box; SURVEY 8e): readout GEMM fused with the
 * reduce-scatter by object.  Each rank multiplies ITS slots; the tile of group g is added (red.add.f32, system scope)
 * straight from the GEMM epilogue into rank_dst[owner[g]] + out_row[g] * ld_out, the fp32 [objects_owned * cv, q]
 * buffer of the rank that owns object g - peer memory mapped through CUDA IPC, or local.  rank_dst: HOST array of
 * n_ranks (<= 8) device pointers.  The caller zeroes the buffers beforehand and fences the ranks afterwards. */
DEVA_B200_API int deva_b200_readout_sparse_scatter(const void* values, int64_t values_ld, int64_t values_rows,
                                                   const int32_t* val_row, const int32_t* out_row,
                                                   const int32_t* owner, int n_groups, int rows_per_group,
                                                   const int32_t* idx, const float* w, int top_k, int n_window, int q,
                                                   void* workspace, float* const* rank_dst, int n_ranks,
                                                   int64_t ld_out, deva_stream_t stream);
/* Peer-visible buffers for the scatter read-out.  peer_alloc: cudaMalloc (zeroed) on `device` + its 64-byte CUDA IPC
 * handle, to be sent to the other ranks; peer_open: map a peer's handle INTO `device`'s address space
 * (cudaIpcOpenMemHandle with lazy peer access - an IPC mapping opened under the exporter's device is not reachable
 * from other devices); peer_close / peer_free undo them. */
DEVA_B200_API int deva_b200_peer_alloc(int device, int64_t bytes, void** ptr, uint8_t handle[64]);
DEVA_B200_API int deva_b200_peer_open(int device, const uint8_t handle[64], void** ptr);
DEVA_B200_API int deva_b200_peer_close(int device, void* ptr);
DEVA_B200_API int deva_b200_peer_free(int device, void* ptr);

/* ---- bank compaction (sieve_by_range / remove_obsolete_features, kv_memory_store.py:127-185) ----------
 * dst must not alias src.  idx: device int32 [n]. */
DEVA_B200_API int deva_b200_gather_rows(void* dst, const void* src, const int32_t* idx, int n, int row_bytes, deva_stream_t stream);
DEVA_B200_API int deva_b200_gather_f32(float* dst, const float* src, const int32_t* idx, int n, deva_stream_t stream);
DEVA_B200_API int deva_b200_gather_cols_f16(void* dst, int64_t ld_dst, const void* src, int64_t ld_src, const int32_t* idx,
                              int rows, int n, deva_stream_t stream);
/* usage[i] = use_cnt[i] / life_cnt[i]  (KeyValueMemoryStore.get_usage, kv_memory_store.py:187-193) */
DEVA_B200_API int deva_b200_usage(float* out, const float* use_cnt, const float* life_cnt, int n, deva_stream_t stream);

/* ==== network path: NHWC fp16 implicit-GEMM convolution + helper kernels ===================================
 * Activations are fp16 NHWC [batch, h, w, c] with c a multiple of 64 (8 for the helpers); weights are packed
 * fp16 [cout_pad, kh*kw*cin_pad] (filter tap major, input channel minor), bias fp32 [cout_pad] with the
 * eval-mode BatchNorm already folded in. */
typedef struct deva_b200_conv_desc {
  const void* x;        /* fp16 NHWC input [batch, h, w, cin_pad] */
  const void* x2;       /* optional second input of the same shape: the convolution sees cat[x, x2] along channels
                         * (weights packed [cout_pad, 2, kh*kw, cin_pad]); stride 1 only */
  const void* x_lo;     /* optional fp16 low-order part of x (x_true = x + x_lo): split-precision mode
                         * D = Xh.Wh + Xl.Wh + Xh.Wl with weights packed [cout_pad, 2 (hi, lo), kh*kw, cin_pad];
                         * ~fp32 accuracy at 3x the MMA work.  Exclusive with x2. */
  int32_t split_mode;   /* 0: as described above (x_lo => three passes);  2: no x_lo, weights packed (hi, lo) as for
                         * mode 0, D = X.Wh + X.Wl (removes the weight rounding);  3: see x_lo8 below */
  int32_t batch, h, w, cin_pad;
  const void* w_packed; /* fp16 [cout_pad, kh*kw*cin_pad] */
  int32_t kh, kw, stride; /* 1x1 or 3x3, stride 1 or 2, padding kh/2 (nn.Conv2d semantics) */
  int32_t cout, cout_pad, nt; /* real / padded output channels, channel tile (multiple of 32, <= 256, divides cout_pad) */
  int32_t th, tw;       /* spatial tile of the implicit GEMM: a th x tw rectangle with th*tw == 128, or th = 0, tw = 128
                         * for flat tiles (stride 1, no out_pool4): output pixels 128t .. 128t+127 of one image in
                         * row-major order, so that no MMA row is spent on padding where no rectangle fits ho x wo */
  const float* bias;
  const void* res;      /* optional fp16 NHWC residual added before the activation (shape of the output) */
  const void* res_lo;   /* optional low-order part of the residual */
  int32_t res_broadcast; /* 1: `res` is ONE image broadcast over the batch */
  const float* rank1_w; /* optional fp32 [cout_pad]: weight of an extra 1-channel input ... */
  const float* rank1_x; /* ... whose fp32 plane is [batch, ho*wo]  (out += rank1_w[c] * rank1_x[b, pixel]) */
  void* out_raw;        /* optional fp16 NHWC output */
  void* out_relu;       /* optional fp16 NHWC output, ReLU applied */
  float* out_f32;       /* optional fp32 NHWC output */
  void* out_raw_lo;     /* optional fp16 remainders (value - fp16(value)) of out_raw / out_relu */
  void* out_relu_lo;
  const float* head_w;  /* optional fused 1x1 head on the ReLU'd fp32 result (needs cout == cout_pad == nt, one of 64 / 128 / 192 / 256): fp32 [head_n, cout] */
  float* head_out;      /* fp32 [batch*ho*wo, head_n]: head_out[p, t] = sum_c relu(out[p, c]) * head_w[t, c] */
  int32_t head_n;       /* <= 9.  Folds MaskDecoder.pred (big_modules.py:189-190) into the last decoder conv. */
  /* optional fused gate epilogue (SensoryUpdater / SensoryDeepUpdater, modules.py:145-149,163-167): the conv output is
   * never written; with C = cout/3 hidden channels the channel tile (nt must be 192) holds [forget | update | new] x 64
   * for hidden channels 64*tile .. +63 (weight rows / bias packed in that order) and the epilogue writes
   * gate_out = sigmoid(f) * gate_h * (1 - sigmoid(u)) + sigmoid(u) * tanh(n), evaluated on the fp32 accumulators. */
  const void* gate_h;   /* fp16 NHWC [batch, ho, wo, cout/3] previous hidden state */
  void* gate_out;       /* fp16 NHWC [batch, ho, wo, cout/3] new hidden state */
  /* split_mode 3: a low-order activation pass on the fp8 tensor-core path (removes the activation-operand rounding at
   * half the cost of a second fp16 pass):
   * D = (X . W16 + Xlo8 . W8) * acc_scale, W16 = fp16(W * 2^S) in w_packed, W8 = e4m3(W * 2^(S-12)) in w8_packed,
   * Xlo8 = e4m3((x - fp16(x)) * 4096) in x_lo8, acc_scale = 2^-S.  Stride 1, cin_pad % 128 == 0. */
  const void* x_lo8;    /* u8 NHWC [batch, h, w, cin_pad] */
  const void* w8_packed; /* u8 [cout_pad, kh*kw*cin_pad] */
  float acc_scale;      /* 0 = 1 */
  void* out_relu_lo8;   /* optional u8 NHWC: e4m3 low-order part (x 4096) of the ReLU'd output */
  int32_t ksplit;       /* > 1: split the K loop into that many chains (fp32 output only): out_f32 then holds
                         * ceil(k_iters / ceil(k_iters / ksplit)) partial sums [part, batch, ho, wo, cout] (bias in part 0)
                         * for the consumer to add in fp32.  The tensor core's accumulator rounds toward zero at every
                         * accumulation step; short chains keep a split-precision convolution at fp32 accuracy. */
  void* out_pool4;      /* optional fp16 NHWC [batch, ho/4, wo/4, cout]: 4x4 average of the raw (pre-ReLU) fp16 output,
                         * equal to deva_b200_area_down(out_raw, 4) bit for bit.  Needs the staged epilogue (every channel
                         * tile exactly 64 / 128 / 192 / 256 wide and cout == cout_pad, no fp32 output, no split-K), tile
                         * sides th, tw and output sides ho, wo multiples of 4; other launches are refused. */
} deva_b200_conv_desc;
/* nn.Conv2d + folded BatchNorm (+ residual, + ReLU) as in deva/model/resnet.py:46-114, group_modules.py:41-67,
 * modules.py:22-39; `desc` is a HOST struct. */
DEVA_B200_API int deva_b200_conv2d(const deva_b200_conv_desc* desc, deva_stream_t stream);
/* im2col of the 7x7 stride-2 pad-3 stems (resnet.py:120): src fp32 planes [b, c, h, w] -> fp16 [b, h/2, w/2, k_pad],
 * column (kh*7+kw)*c + ch, zero padded to k_pad (multiple of 64).  The stem then runs through deva_b200_conv2d as a
 * 1x1 convolution over k_pad channels.  dst_lo (optional) receives the fp16 remainders for split precision. */
DEVA_B200_API int deva_b200_stem_im2col(const float* src, void* dst, void* dst_lo, int b, int c, int h, int w, int k_pad,
                                        deva_stream_t stream);
DEVA_B200_API int deva_b200_nchw_to_nhwc(const float* src, void* dst, int b, int c, int h, int w, int c_pad,
                                         deva_stream_t stream);
/* 3x3 stride-2 max pool (resnet.py:123); x_lo / y_lo: optional low-order parts (pooling acts on x + x_lo) */
DEVA_B200_API int deva_b200_maxpool(const void* x, const void* x_lo, void* y, void* y_lo, int b, int h, int w, int c,
                                    deva_stream_t stream);
/* F.interpolate(mode='area') by an integer ratio r (group_modules.py:33-38), fp16 NHWC and fp32 planes */
DEVA_B200_API int deva_b200_area_down(const void* x, void* y, int b, int h, int w, int c, int r, deva_stream_t stream);
DEVA_B200_API int deva_b200_area_down_plane(const float* x, float* y, int b, int h, int w, int r, deva_stream_t stream);
/* Bilinear x2 (align_corners=False) + broadcast skip add (modules.py:88-91) and x + CBAM(x) (cbam.py:21-77 inside
 * group_modules.py:146-150) on a residual stream carried as fp16 (hi, lo) pairs (the "parity" precision plan): the input
 * is g + g_lo + skip + skip_lo (x + x_lo), the raw result is written as (raw, raw_lo), the ReLU'd copy (an MMA operand) as
 * hi.  relu_lo8 (optional): u8 NHWC, e4m3 of (relu - fp16(relu)) * 4096 - the low-order operand of a conv with
 * split_mode 3.  cbam_split takes the gate statistics (channel pooling, per-pixel max / mean) over x + x_lo; scratch: fp32
 * [129*b*c + 2*b*h*w] (2 x 64 pooling slices + the gate, then the per-pixel statistics); c = 8 x a divisor of 256. */
DEVA_B200_API int deva_b200_up2_add_split(const void* g, const void* g_lo, const void* skip, const void* skip_lo,
                                          void* raw, void* raw_lo, void* relu, void* relu_lo8, int b, int h, int w, int c,
                                          deva_stream_t stream);
DEVA_B200_API int deva_b200_cbam_split(const void* x, const void* x_lo, const float* w1, const float* b1, const float* w2,
                                       const float* b2, const float* ws, const float* bs, float* scratch, void* raw,
                                       void* raw_lo, void* relu, int b, int h, int w, int c, int r, deva_stream_t stream);
/* Finish of a split-K convolution (deva_b200_conv2d with ksplit > 1): out = sum of the n_parts fp32 partial sums
 * (part_stride elements apart, bias in part 0) + optional fp16 residual (res + res_lo), written as fp16 raw / ReLU'd
 * tensors, each optionally as a (hi, lo) pair.  n = elements per part (multiple of 8). */
DEVA_B200_API int deva_b200_sum_parts(const float* parts, int n_parts, int64_t part_stride, const void* res,
                                      const void* res_lo, void* raw, void* raw_lo, void* relu, void* relu_lo, int64_t n,
                                      deva_stream_t stream);
/* key projection tail (modules.py:73-78): y fp32 [q, ld] = [key | d | e], given as n_parts partial sums part_stride
 * elements apart (deva_b200_conv2d's ksplit) -> key [q,ck], shrinkage [q] = d^2 + 1, selection [q,ck] = sigmoid(e) */
DEVA_B200_API int deva_b200_key_tail(const float* y, int ld, int q, int ck, int n_parts, int64_t part_stride, float* key,
                                     float* shrinkage, float* selection, deva_stream_t stream);
/* sigmoid -> aggregate -> bilinear x4 -> softmax (network.py:33-40,144-168): logits fp32 [k,h,w] ->
 * prob fp32 [(k+1),4h,4w] (and optionally the up-sampled logits); agg: fp32 scratch [(k+1),h,w] */
DEVA_B200_API int deva_b200_output_tail(const float* logits, float* agg, float* prob, float* logits_out, int k, int h,
                                        int w, deva_stream_t stream);
/* logits[b,y,x] = bias + sum_{dy,dx} z[b, y+dy, x+dx, (dy+1)*3+(dx+1)]: the 3x3 gather completing the fused head
 * (z fp32 [b,h,w,9] from deva_b200_conv2d's head_out) == nn.Conv2d(256, 1, 3, padding=1) on relu(p4) */
DEVA_B200_API int deva_b200_head_gather3x3(const float* z, float* out, float bias, int b, int h, int w,
                                           deva_stream_t stream);
/* fp16 token-major values [n, c] -> bank rows dst[c, j] (ld_dst): append from the NHWC value encoder */
DEVA_B200_API int deva_b200_transpose_append(const void* src, void* dst, int64_t ld_dst, int n, int c,
                                             deva_stream_t stream);

/* ---- frame ingest / egress (SURVEY 8f-3) ------------------------------------------------------------------------ */
/* Decoded frame u8 [h, w, 3] (RGB interleaved) -> fp32 [3, h, w], (x / 255 - mean[c]) / std[c]: torchvision's
 * ToTensor + Normalize (deva/inference/data/video_reader.py:146-150) after the upload instead of before it (4x fewer
 * PCIe bytes).  Bit-exact with the torch ops (IEEE divisions in the same order). */
DEVA_B200_API int deva_b200_ingest_rgb8(const uint8_t* src, float* dst, int h, int w, const float mean[3],
                                        const float std[3], deva_stream_t stream);
/* Decoded frame u8 [h, w, 3] -> fp32 [3, out_h, out_w]: ToTensor + Normalize of every source pixel exactly as
 * deva_b200_ingest_rgb8, then a separable resample - horizontal into scratch fp32 [3, h, out_w], then vertical - and an
 * optional horizontal flip of the result.  Output pixel o of an axis is sum_{j < taps} w[o * taps + j] * in[idx[o * taps
 * + j]] (fused multiply-adds in ascending j); the int32 idx / fp32 w tables of each axis come from the caller (the
 * package builds them from torch's CPU bilinear and antialiased-bilinear arithmetic: video_reader.py:151's
 * Resize(BILINEAR, antialias=True) and demo_utils.py:18's F.interpolate(mode='bilinear')). */
DEVA_B200_API int deva_b200_ingest_rgb8_resize(const uint8_t* src, int h, int w, int out_h, int out_w,
                                               const int32_t* x_idx, const float* x_w, int x_taps, const int32_t* y_idx,
                                               const float* y_w, int y_taps, float* scratch, float* dst, int flip,
                                               const float mean[3], const float std[3], deva_stream_t stream);
/* Index mask u8 [h, w] -> int64 [out_h, out_w]: dst[y, x] = src[y_idx[y], x_idx[x']], x' = out_w - 1 - x when flip,
 * else x.  With PIL's NEAREST index maps this is the reader's Resize(NEAREST) of a first-frame mask
 * (video_reader.py:159-161), then eval_vos.py:162-164's flip. */
DEVA_B200_API int deva_b200_mask_nearest(const uint8_t* src, int h, int w, int out_h, int out_w, const int32_t* x_idx,
                                         const int32_t* y_idx, int flip, int64_t* dst, deva_stream_t stream);
/* Mask u8 [h, w, channels] (channels 1 or 3) -> int32 [out_h, out_w] through the same gather as deva_b200_mask_nearest:
 * one channel gives the index, three give the RGB id r + 256 g + 65536 b.  With PIL's NEAREST index maps this is the
 * detection reader's Resize(NEAREST) of a P / L / RGB mask and its np.array(..., dtype=np.int32) id map
 * (detection_video_reader.py:99-106). */
DEVA_B200_API int deva_b200_mask_nearest_ids(const uint8_t* src, int channels, int h, int w, int out_h, int out_w,
                                             const int32_t* x_idx, const int32_t* y_idx, int flip, int32_t* dst,
                                             deva_stream_t stream);
/* Pillow's Image.resize((out_w, out_h), BILINEAR) of k 8-bit one-channel planes src u8 [k, h, w], written as float32
 * v / 255 into dst [k, out_h, out_w] (the reader's soft mask, video_reader.py:188-191).  Per axis, bounds int32
 * [n_out, 2] (first input index, taps) and coef int32 [n_out, taps] are libImaging's precompute_coeffs and
 * normalize_coeffs_8bpc (22-bit fixed point); the horizontal pass runs first and rounds to u8 in scratch u8
 * [k, h, out_w], then the vertical pass.  A pass whose axis keeps its size is skipped (its tables may be NULL); scratch
 * is needed only when both run. */
DEVA_B200_API int deva_b200_pil_resample_u8(const uint8_t* src, int k, int h, int w, int out_h, int out_w,
                                            const int32_t* x_bounds, const int32_t* x_coef, int x_taps,
                                            const int32_t* y_bounds, const int32_t* y_coef, int y_taps, uint8_t* scratch,
                                            float* dst, deva_stream_t stream);
/* Driver post-step (evaluation/eval_vos.py:169-181) in one pass: optional bilinear resize (align_corners=False) of
 * prob fp32 [c, h, w] to [out_h, out_w], optional horizontal flip, argmax over channels (first maximum wins),
 * temporary-id -> object-id remap through lut int32 [c] (lut[0] = 0).  Writes out_u8 [out_h, out_w] and/or
 * out_i64 [out_h, out_w] (either may be NULL). */
DEVA_B200_API int deva_b200_prob_to_ids(const float* prob, int c, int h, int w, int out_h, int out_w, int flip,
                                        const int32_t* lut, uint8_t* out_u8, int64_t* out_i64, deva_stream_t stream);
/* Result-saver egress (deva/inference/result_utils.py:98-102 and the per-frame work of save_result, :158-257) in one
 * pass: the resize and argmax of deva_b200_prob_to_ids without flip (its id map, bit for bit), then per output pixel of
 * argmax channel k, each output optional (NULL = not written):
 *  - out_u8 [out_h, out_w] = (uint8)lut[k]: the remapped index mask (:159-163, :217);
 *  - out_rgb [out_h, out_w, 3] = bytes (v & 255, v >> 8 & 255, v >> 16 & 255) of v = rgb[k]: the long-id RGB image
 *    (:208-215; the caller packs ID2RGBConverter._id_to_rgb(id) for the ids it colours, 0 for the others);
 *  - out_overlay [out_h, out_w, 3] = frame where lut[k] == 0, else (frame + id image) >> 1: the visualisation blend
 *    (:240-242; frame u8 [out_h, out_w, 3]);
 *  - counts int64 [c] (pixels per channel) and boxes int32 [c, 4] (x_min, y_min, x_max, y_max; (INT32_MAX, INT32_MAX,
 *    -1, -1) for an empty channel), written together: the segment areas (:166-171, :198-204) and masks_to_boxes
 *    (:244-257).  The call initialises them.
 * lut int32 [c] is required; rgb uint32 [c] with out_rgb or out_overlay.  c <= DEVA_B200_MAX_SEGMENT_CHANNELS. */
DEVA_B200_API int deva_b200_prob_to_segments(const float* prob, int c, int h, int w, int out_h, int out_w,
                                             const int32_t* lut, const uint32_t* rgb, const uint8_t* frame,
                                             uint8_t* out_u8, uint8_t* out_rgb, uint8_t* out_overlay, int64_t* counts,
                                             int32_t* boxes, deva_stream_t stream);
/* Score export of multi-scale / flip evaluation (evaluation/eval_vos.py:169-177 with --save_scores, :188-189): the
 * resize and flip of deva_b200_prob_to_ids (the same values, bit for bit), then per channel and output pixel
 * s = (uint8)(v * 255) with one round-to-nearest float multiply and truncation, numpy's (x * 255).astype(np.uint8) on
 * float32.  Each output optional, at least one given: scores u8 [c, out_h, out_w] = s; sum int32 [c, out_h, out_w] += s
 * (the running sum of scripts/merge_multi_scale.py). */
DEVA_B200_API int deva_b200_prob_to_scores(const float* prob, int c, int h, int w, int out_h, int out_w, int flip,
                                           uint8_t* scores, int32_t* sum, deva_stream_t stream);
/* Merge of multi-scale / flip scores (scripts/merge_multi_scale.py:process_vid): the channel of the first maximum of
 * sum int32 [c, h, w] (np.argmax's tie order), mapped through lut int32 [c] (NULL: the channel itself).  Writes out_u8
 * [h, w] and/or out_i64 [h, w] (either may be NULL, not both). */
DEVA_B200_API int deva_b200_scores_to_ids(const int32_t* sum, int c, int h, int w, const int32_t* lut, uint8_t* out_u8,
                                          int64_t* out_i64, deva_stream_t stream);


/* ---- video panoptic metrics (deva/vps_metrics) -------------------------------------------------------------------
 * Frames are RGB id images u8 [h, w, 3] with id = r + 256 g + 65536 b (the VIPSeg PNG encoding).  An id table is a
 * sorted int32 array; a pixel's index is the position of its id in the table, or n (the table's length) when the id is
 * not in it.  The tables live in shared memory: n_gt + n_pred (n_table + n_out) entries take at most 200 KiB.
 *
 * Joint label histogram of one ground-truth and one predicted frame, from which VPQ's intersections and areas
 * (deva/vps_metrics/eval_vpq_vipseg.py:106-257) and STQ's confusion, tube areas and intersections
 * (eval_stq_vipseg.py:123-151, segmentation_and_tracking_quality.py:111-195) are regroupings of cells:
 * hist int32 [n_gt + 1, n_pred + 1], cell (i, j) = pixels whose gt index is i and pred index is j.  The call initialises
 * hist.  A histogram that fits in shared memory next to the tables is kept per block there; a larger one is counted
 * with global atomics. */
DEVA_B200_API int deva_b200_pano_joint_hist(const uint8_t* gt, const uint8_t* pred, int h, int w, const int32_t* gt_ids,
                                            int n_gt, const int32_t* pred_ids, int n_pred, int32_t* hist,
                                            deva_stream_t stream);
/* Stuff merging's id rewrite (deva/vps_metrics/stuff_merging.py:45-83): a pixel of pred index i takes the id
 * out_ids[slot[i]] (slot int32 [n_table + 1]; slot[n_table] for ids not in the table), written to out u8 [h, w, 3] as
 * bytes (id >> 8k) & 255.  counts int32 [n_out]: pixels written per slot; unknown int32 [1]: pixels whose id is not in the
 * table.  The call initialises counts and unknown. */
DEVA_B200_API int deva_b200_pano_remap(const uint8_t* pred, int h, int w, const int32_t* ids, int n_table,
                                       const int32_t* slot, const int32_t* out_ids, int n_out, uint8_t* out,
                                       int32_t* counts, int32_t* unknown, deva_stream_t stream);

/* ---- label statistics and rewrite (deva/inference/postprocess_unsup_davis17.py) ----------------------------------
 * A frame is u8 [h, w, channels] with channels 1 (the label is the byte: a P or L image) or 3 / 4 (the label is
 * r << 16 | g << 8 | b, alpha ignored: postprocess_unsup_davis17.py:22-24).  Label 0 is background.
 *
 * Pixel count of every non-zero label of one frame.  labels / counts int32 [capacity] are the call's open-addressed table
 * and then its result: once the work completes, state[0] = n and labels[0, n) / counts[0, n) are the frame's n distinct
 * non-zero labels and their pixel counts, in no particular order.  If the frame has more than `capacity` distinct
 * non-zero labels, state[0] = -1 and the lists are not valid: since the call does not synchronise, a capacity overflow
 * is reported there, and the caller must check state[0] before it uses the lists (deva/_native.py raises).  state int32
 * [2] (state[1] is scratch).  The call initialises all three. */
DEVA_B200_API int deva_b200_label_areas(const uint8_t* frame, int h, int w, int channels, int capacity, int32_t* labels,
                                        int32_t* counts, int32_t* state, deva_stream_t stream);
/* out u8 [h, w]: (uint8)index[i] for a pixel whose label is labels[i], 0 for a label not in the table.  labels int32 [n]
 * sorted ascending (distinct), index int32 [n]; 2 n entries take at most 200 KiB (shared memory). */
DEVA_B200_API int deva_b200_label_to_index(const uint8_t* frame, int h, int w, int channels, const int32_t* labels,
                                           const int32_t* index, int n, uint8_t* out, deva_stream_t stream);

/* ---- detector masks -> detection id map (deva/ext/automatic_sam.py auto_segment, deva/ext/grounding_dino.py
 * segment_with_text) ------------------------------------------------------------------------------------------------
 * masks u8 [n, h, w] (a bool or uint8 mask stack's bytes).  Mask k's value v_k at an output pixel of [out_h, out_w] is
 * the bilinear resize (align_corners = False, F.interpolate's arithmetic; a copy when the sizes are equal) of the bytes
 * as floats.  Any n >= 0; per-mask counters live in shared memory up to DEVA_B200_MASK_SMEM_COUNTERS, in global memory
 * beyond.  The calls initialise their outputs.
 *
 * area float [n]: fp32 sum of v_k over the output, deterministic (fixed partial slots added in a fixed order, no float
 * atomics: equal masks get equal areas).  covered int32 [n]: pixels with v_k > 0.5.  Either may be null.  workspace:
 * deva_b200_mask_stats_workspace_bytes(n, out_h, out_w) bytes. */
DEVA_B200_API size_t deva_b200_mask_stats_workspace_bytes(int n, int out_h, int out_w);
DEVA_B200_API int deva_b200_mask_stats(const uint8_t* masks, int n, int h, int w, int out_h, int out_w, void* workspace,
                                       float* area, int32_t* covered, deva_stream_t stream);
/* slot int32 [out_h, out_w]: slot of the first maximum of [0.1, v_0 * score[0], ..., v_{n-1} * score[n-1]] (0 = the
 * 0.1 background, k + 1 = mask k); with kept_only, 0 wherever the winner's v < 0.5.  won / kept int32 [n + 1]: pixels
 * each slot wins / wins with v >= 0.5.  score float [n]. */
DEVA_B200_API int deva_b200_mask_scored_argmax(const uint8_t* masks, int n, int h, int w, int out_h, int out_w,
                                               const float* score, int kept_only, int32_t* slot, int32_t* won,
                                               int32_t* kept, deva_stream_t stream);
/* slot int32 [out_h, out_w]: k + 1 for the last mask k of order int32 [n] (a permutation of 0..n-1, the paint order)
 * with v_k > 0.5, 0 where there is none.  covered int32 [n]: pixels with v_k > 0.5, indexed by mask. */
DEVA_B200_API int deva_b200_mask_last_cover(const uint8_t* masks, int n, int h, int w, int out_h, int out_w,
                                            const int32_t* order, int32_t* slot, int32_t* covered,
                                            deva_stream_t stream);

/* ---- PNG image data (deva/utils/png_encode.py; the format is DESIGN §7) ------------------------------------------
 * img u8 [h, w] (channels 1: an L or P image, at bits 1, 2, 4 or 8) or [h, w, 3] (channels 3, bits 8).  Writes the zlib
 * stream of the PNG's IDAT to out and its byte length to out_len (int64 [1]), both on the device; the chunks around it
 * are the caller's.  Rows are Up-filtered, tokenised greedily at distances 1 and bytes-per-pixel and coded with
 * deflate's fixed Huffman codes, so the bytes are a function of the image alone.  out: deva_b200_png_bound(h, w,
 * channels, bits) bytes (every filtered byte a 9-bit literal, rounded up to 4 bytes), 4-byte aligned; workspace:
 * deva_b200_png_workspace_bytes(h) bytes, 8-byte aligned.  A row's bytes + 5 must fit in a block's shared memory. */
DEVA_B200_API size_t deva_b200_png_bound(int h, int w, int channels, int bits);
DEVA_B200_API size_t deva_b200_png_workspace_bytes(int h);
DEVA_B200_API int deva_b200_png_encode(const uint8_t* img, int h, int w, int channels, int bits, void* workspace,
                                       uint8_t* out, int64_t* out_len, deva_stream_t stream);

/* ---- baseline JPEG scan (deva/utils/jpeg_encode.py; the format is DESIGN §7) --------------------------------------
 * img u8 [h, w, 3] RGB, 1 <= h, w <= 65535.  Writes the entropy-coded segment of a baseline 4:2:0 JPEG followed by EOI
 * to out and its byte length to out_len (int64 [1]), both on the device; the marker segments before it (SOI .. SOS) are
 * the caller's.  The arithmetic is libjpeg's (jccolor.c colour, h2v2 downsampling with libjpeg's edge padding, islow
 * DCT, rounding quantisation, Annex K Huffman tables, 1-bit fill, 0x00 after every 0xFF), so the bytes are a function of
 * the image and the tables alone and equal Pillow's default save.  quality_tables: HOST, 64 luma then 64 chroma
 * quantisation values in zigzag order, each in [1, 255].  out: deva_b200_jpeg_bound(h, w) bytes (every block at its
 * worst case, every byte stuffed, plus EOI); workspace: deva_b200_jpeg_workspace_bytes(h, w) bytes, 16-byte aligned. */
DEVA_B200_API size_t deva_b200_jpeg_bound(int h, int w);
DEVA_B200_API size_t deva_b200_jpeg_workspace_bytes(int h, int w);
DEVA_B200_API int deva_b200_jpeg_encode(const uint8_t* img, int h, int w, const uint8_t* quality_tables, void* workspace,
                                        uint8_t* out, int64_t* out_len, deva_stream_t stream);

/* ---- COCO compressed RLE (deva/utils/rle_encode.py; the format is DESIGN §7) --------------------------------------
 * ids i64 [h, w] row-major, 1 <= h, w and h * w < 2^31; seg_ids i64 [n], 1 <= n <= DEVA_B200_MAX_SEGMENT_CHANNELS, both
 * on the device.  For every j < n, out[offsets[j] : offsets[j + 1]] is the counts string pycocotools' rleToString
 * writes for the column-major RLE of the mask ids == seg_ids[j]; offsets: i64 [n + 1] on the device, offsets[0] = 0.  A
 * repeated seg id gets the same string again; an id absent from the map gets the string of [h * w].  The bytes are a
 * function of the inputs alone.  out: deva_b200_rle_bound(h, w, n) bytes = n * (h * w + 1), the longest string (a mask
 * that changes at every pixel) for every entry; workspace: deva_b200_rle_workspace_bytes(h, w, n) bytes, 16-byte
 * aligned.  Neither depends on the map's content. */
DEVA_B200_API size_t deva_b200_rle_bound(int h, int w, int n);
DEVA_B200_API size_t deva_b200_rle_workspace_bytes(int h, int w, int n);
DEVA_B200_API int deva_b200_rle_encode(const int64_t* ids, int h, int w, const int64_t* seg_ids, int n, void* workspace,
                                       uint8_t* out, int64_t* offsets, deva_stream_t stream);

/* ---- PNG decode (deva/utils/png_decode.py; the format rules are DESIGN §7) ----------------------------------------
 * A batch of n files: streams holds their zlib streams (the concatenated IDAT data of each), desc int64 [n, 8] per file
 * {stream offset, stream length, h, w, colour type, bit depth, output offset, workspace offset}, all on the device.  A
 * supported file is grey at 2, 4 or 8 bits, palette at 1, 2, 4 or 8, RGB 8 or RGBA 8, non-interlaced.  For each file
 * whose stream is one well-formed zlib stream that inflates to exactly h * (rowbytes + 1) bytes with a matching
 * Adler-32, nothing after it, and every row's filter type <= 4, out[output offset ..] receives Pillow's array ([h, w]
 * or [h, w, 3 | 4] uint8; 2- and 4-bit grey scaled by 85 and 17, palette indices unscaled) and status[i] = 0; any other
 * file gets a nonzero int32 status and its output bytes are undefined.  Every read of a stream is bounded by its length
 * and every write by the file's shape.  workspace + workspace offset: deva_b200_png_decode_workspace_bytes(h, w, colour
 * type, bit depth) bytes per file (its filtered stream), 0 for an unsupported shape.  Enqueued on stream without
 * synchronising the host; allocates nothing. */
DEVA_B200_API size_t deva_b200_png_decode_workspace_bytes(int h, int w, int colour_type, int bits);
DEVA_B200_API int deva_b200_png_decode(const uint8_t* streams, const int64_t* desc, int n, uint8_t* out, void* workspace,
                                       int32_t* status, deva_stream_t stream);

/* ---- JPEG decode (deva/utils/jpeg_decode.py; the format rules are DESIGN §7) ---------------------------------------
 * A batch of n baseline files, all on the device: scans holds their entropy-coded data with the stuffing bytes and
 * RSTn markers removed; desc int64 [n, 11] per file {scan offset, scan length, h, w, luma h sampling, luma v sampling,
 * tables index, output offset, workspace offset, first subsequence, subsequences}; tables int32 [n, 5016] per file (the
 * DC and AC Huffman lookups of each component and its quantisation table in natural order, csrc/jpeg_decode.cuh);
 * intervals int64 [n_intervals, 6] per restart interval {file, bit start, bit end, first block, blocks, first
 * subsequence}; subs int64 [n_subs, 3] per subsequence {interval, bit start, bit end}, the subsequences of an interval
 * consecutive and covering it, bits counted from scans.  Y is sampled 1x1, 2x1 or 2x2 and Cb, Cr 1x1.  For each file
 * whose every interval decodes to exactly its blocks, with at most 7 padding bits left, every code in its table,
 * categories <= 11 (DC) and 10 (AC), no run past coefficient 63, and every block in the range where libjpeg-turbo's C
 * and x86 SIMD islow IDCTs agree, out[output offset ..] receives Pillow's array ([h, w, 3] uint8: islow IDCT, fancy
 * upsampling, jdcolor.c's YCbCr -> RGB) and status[i] = 0; any other file gets a nonzero int32 status and undefined
 * output bytes.  Every read of the scans is bounded by its interval and every write by the file's shape.  workspace:
 * deva_b200_jpeg_decode_workspace_bytes(0, 0, 0, 0, 0) bytes shared by the batch (its int32 word 3 receives the number
 * of synchronisation rounds), then at each file's workspace offset deva_b200_jpeg_decode_workspace_bytes(h, w, luma h,
 * luma v, subsequences) bytes (0 for an unsupported shape).  The entropy decode is one cooperative launch.  Enqueued on
 * stream without synchronising the host; allocates nothing. */
DEVA_B200_API size_t deva_b200_jpeg_decode_workspace_bytes(int h, int w, int luma_h, int luma_v,
                                                           int64_t subsequences);
DEVA_B200_API int deva_b200_jpeg_decode(const uint8_t* scans, const int64_t* desc, int n, const int32_t* tables,
                                        const int64_t* intervals, int64_t n_intervals, const int64_t* subs,
                                        int64_t n_subs, uint8_t* out, void* workspace, int32_t* status,
                                        deva_stream_t stream);

/* ---- Segment Anything automatic masks (deva/ext/sam_masks.py; DESIGN §7) -------------------------------------------
 * logits fp32 [n, lh, lw] contiguous: the mask decoder's low-resolution logits.  Every value below is Sam.postprocess_masks'
 * float32 value at a frame pixel: torch's CUDA bilinear upsample (align_corners=False) of the logits to [grid, grid],
 * cropped to [in_h, in_w], then the same upsample to [out_h, out_w].  1 <= in_h, in_w <= grid <= 1024, out_h * out_w
 * < 2^31; n <= 65535.
 * sam_mask_stats: stats int32 [n, 7] per mask {pixels > thr_hi, > thr_lo, > thr, x0, y0, x1, y1}, the box being the
 * extent of the pixels > thr (x1 = y1 = -1 when there are none).  With iou (fp32 [n], optional), a mask whose
 * iou > iou_thresh fails is not evaluated and its counts stay 0.
 * sam_mask_compact: one CTA.  stability[i] = float(count > thr_hi) / float(count > thr_lo) (nan for 0 / 0); boxes i64
 * [n, 4] = {x0, y0, x1, y1}, or zeros for a mask with no pixel > thr; kept int32 [n + 1]: kept[0] = the number of masks
 * with iou > iou_thresh (when iou is given) and stability >= stability_thresh (when stability_thresh > 0), then their
 * indices in ascending order.
 * sam_nms: torchvision's CUDA nms of boxes fp32 [n, 4] (x0, y0, x1, y1) by scores fp32 [n]: a stable descending sort of
 * the scores, IoU = inter / (area_a + area_b - inter) in float32, a box suppressed when its IoU with a kept box of
 * higher rank is > iou_thresh.  keep i64 [n]: the kept indices in rank order, the first *n_keep valid.  workspace:
 * deva_b200_sam_nms_workspace_bytes(n) bytes, 16-byte aligned.
 * sam_mask_write: out bool [n, out_h, out_w]: mask m is the value of logits[sel[m]] > thr (sel i64 [n]). */
DEVA_B200_API int deva_b200_sam_mask_stats(const float* logits, int n, int lh, int lw, int grid, int in_h, int in_w,
                                           int out_h, int out_w, const float* iou, float iou_thresh, float thr_hi,
                                           float thr_lo, float thr, int32_t* stats, deva_stream_t stream);
DEVA_B200_API int deva_b200_sam_mask_compact(const int32_t* stats, const float* iou, int n, float iou_thresh,
                                             float stability_thresh, float* stability, int64_t* boxes, int32_t* kept,
                                             deva_stream_t stream);
DEVA_B200_API size_t deva_b200_sam_nms_workspace_bytes(int n);
DEVA_B200_API int deva_b200_sam_nms(const float* boxes, const float* scores, int n, float iou_thresh, void* workspace,
                                    int64_t* keep, int32_t* n_keep, deva_stream_t stream);
DEVA_B200_API int deva_b200_sam_mask_write(const float* logits, const int64_t* sel, int n, int lh, int lw, int grid,
                                           int in_h, int in_w, int out_h, int out_w, float thr, uint8_t* out,
                                           deva_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DEVA_B200_H_ */
