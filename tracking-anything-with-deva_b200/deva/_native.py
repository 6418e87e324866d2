"""ctypes binding of libdeva_b200.so (C ABI declared in include/deva_b200.h).

This is the only door between the Python host code and the sm_90a kernels.  There is no
fallback: if the library is missing, was built for another ABI version, or a kernel reports an
error, a RuntimeError is raised.  PyTorch is used for device memory and streams only.
"""
import ctypes
import os
from ctypes import c_char_p, c_int, c_int32, c_int64, c_size_t, c_uint64, c_void_p, POINTER

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), 'csrc', 'libdeva_b200.so')
ABI_VERSION = 29
LIST_PITCH = 32
MAX_GROUPS = 256
MAX_SEGMENT_CHANNELS = 8192
MASK_SMEM_COUNTERS = 8192

_lib = None


class ConvDesc(ctypes.Structure):
    """Mirror of ``deva_b200_conv_desc`` (include/deva_b200.h)."""
    _fields_ = [('x', c_void_p), ('x2', c_void_p), ('x_lo', c_void_p), ('split_mode', c_int32), ('batch', c_int32), ('h', c_int32), ('w', c_int32), ('cin_pad', c_int32),
                ('w_packed', c_void_p), ('kh', c_int32), ('kw', c_int32), ('stride', c_int32),
                ('cout', c_int32), ('cout_pad', c_int32), ('nt', c_int32), ('th', c_int32), ('tw', c_int32),
                ('bias', c_void_p), ('res', c_void_p), ('res_lo', c_void_p), ('res_broadcast', c_int32),
                ('rank1_w', c_void_p), ('rank1_x', c_void_p),
                ('out_raw', c_void_p), ('out_relu', c_void_p), ('out_f32', c_void_p),
                ('out_raw_lo', c_void_p), ('out_relu_lo', c_void_p),
                ('head_w', c_void_p), ('head_out', c_void_p), ('head_n', c_int32),
                ('gate_h', c_void_p), ('gate_out', c_void_p), ('x_lo8', c_void_p), ('w8_packed', c_void_p),
                ('acc_scale', ctypes.c_float), ('out_relu_lo8', c_void_p), ('ksplit', c_int32), ('out_pool4', c_void_p)]


_SIGNATURES = {
    'deva_b200_abi_version': (c_int, []),
    'deva_b200_last_error': (c_char_p, []),
    'deva_b200_launch_count': (c_uint64, []),
    'deva_b200_device_check': (c_int, []),
    'deva_b200_pack_query': (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p,
                                     c_void_p, c_void_p]),
    'deva_b200_pack_keys': (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_append_values': (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_void_p]),
    'deva_b200_simtopk_workspace_bytes': (c_size_t, [c_int]),
    'deva_b200_sim_topk': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                   c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p,
                                   c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_merge_lists': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                      c_void_p]),
    'deva_b200_sim_topk_wide_workspace_bytes': (c_size_t, [c_int, c_int]),
    'deva_b200_sim_topk_wide': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                        c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int64, c_void_p,
                                        c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    'deva_b200_merge_lists_wide': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                           c_void_p, c_void_p]),
    'deva_b200_sim_dense_softmax': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                            c_void_p, c_int, c_int, c_void_p, c_int64, c_void_p, c_int64, c_void_p,
                                            c_void_p]),
    'deva_b200_readout': (c_int, [c_void_p, c_int64, c_int64, POINTER(c_int32), POINTER(c_int32), c_int, c_int,
                                  c_void_p, c_int64, c_int, c_int, c_void_p, c_int64, c_void_p, c_void_p]),
    'deva_b200_readout_sparse_workspace_bytes': (c_size_t, [c_int, c_int]),
    'deva_b200_readout_sparse': (c_int, [c_void_p, c_int64, c_int64, POINTER(c_int32), POINTER(c_int32), c_int, c_int,
                                         c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int64, c_void_p,
                                         c_void_p]),
    'deva_b200_readout_sparse_scatter': (c_int, [c_void_p, c_int64, c_int64, POINTER(c_int32), POINTER(c_int32),
                                                 POINTER(c_int32), c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                                 c_void_p, POINTER(c_void_p), c_int, c_int64, c_void_p]),
    'deva_b200_readout_sparse_wide_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'deva_b200_readout_sparse_wide': (c_int, [c_void_p, c_int64, c_int64, POINTER(c_int32), POINTER(c_int32), c_int,
                                              c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                              c_int64, c_void_p, c_void_p]),
    'deva_b200_readout_sparse_scatter_wide': (c_int, [c_void_p, c_int64, c_int64, POINTER(c_int32), POINTER(c_int32),
                                                      POINTER(c_int32), c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                                                      c_int, c_int, c_void_p, POINTER(c_void_p), c_int, c_int64,
                                                      c_void_p]),
    'deva_b200_peer_alloc': (c_int, [c_int, c_int64, POINTER(c_void_p), c_char_p]),
    'deva_b200_peer_open': (c_int, [c_int, c_char_p, POINTER(c_void_p)]),
    'deva_b200_peer_close': (c_int, [c_int, c_void_p]),
    'deva_b200_peer_free': (c_int, [c_int, c_void_p]),
    'deva_b200_gather_rows': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    'deva_b200_gather_f32': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    'deva_b200_gather_cols_f16': (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int, c_int, c_void_p]),
    'deva_b200_usage': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    'deva_b200_conv2d': (c_int, [POINTER(ConvDesc), c_void_p]),
    'deva_b200_stem_im2col': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    'deva_b200_nchw_to_nhwc': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    'deva_b200_maxpool': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    'deva_b200_area_down': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    'deva_b200_area_down_plane': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    'deva_b200_up2_add_split': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_int, c_int, c_int, c_int, c_void_p]),
    'deva_b200_cbam_split': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                     c_void_p]),
    'deva_b200_sum_parts': (c_int, [c_void_p, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_int64, c_void_p]),
    'deva_b200_key_tail': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_output_tail': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    'deva_b200_head_gather3x3': (c_int, [c_void_p, c_void_p, ctypes.c_float, c_int, c_int, c_int, c_void_p]),
    'deva_b200_transpose_append': (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p]),
    'deva_b200_ingest_rgb8': (c_int, [c_void_p, c_void_p, c_int, c_int, ctypes.POINTER(ctypes.c_float),
                                      ctypes.POINTER(ctypes.c_float), c_void_p]),
    'deva_b200_ingest_rgb8_resize': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                             c_void_p, c_int, c_void_p, c_void_p, c_int, ctypes.POINTER(ctypes.c_float),
                                             ctypes.POINTER(ctypes.c_float), c_void_p]),
    'deva_b200_mask_nearest': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                       c_void_p]),
    'deva_b200_mask_nearest_ids': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                           c_void_p, c_void_p]),
    'deva_b200_pil_resample_u8': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                          c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    'deva_b200_prob_to_ids': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                      c_void_p]),
    'deva_b200_prob_to_segments': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_prob_to_scores': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                         c_void_p]),
    'deva_b200_scores_to_ids': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_pano_joint_hist': (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p,
                                          c_void_p]),
    'deva_b200_pano_remap': (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                     c_void_p, c_void_p, c_void_p]),
    'deva_b200_label_areas': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_label_to_index': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                         c_void_p]),
    'deva_b200_mask_stats_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'deva_b200_mask_stats': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                     c_void_p]),
    'deva_b200_mask_scored_argmax': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p,
                                             c_void_p, c_void_p, c_void_p]),
    'deva_b200_mask_last_cover': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                          c_void_p]),
    'deva_b200_png_bound': (c_size_t, [c_int, c_int, c_int, c_int]),
    'deva_b200_png_workspace_bytes': (c_size_t, [c_int]),
    'deva_b200_png_encode': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_jpeg_bound': (c_size_t, [c_int, c_int]),
    'deva_b200_jpeg_workspace_bytes': (c_size_t, [c_int, c_int]),
    'deva_b200_jpeg_encode': (c_int, [c_void_p, c_int, c_int, c_char_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_rle_bound': (c_size_t, [c_int, c_int, c_int]),
    'deva_b200_rle_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'deva_b200_rle_encode': (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_png_decode_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'deva_b200_png_decode': (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_jpeg_decode_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int, c_int64]),
    'deva_b200_jpeg_decode': (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int64, c_void_p,
                                      c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_sam_mask_stats': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                         ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, c_void_p,
                                         c_void_p]),
    'deva_b200_sam_mask_compact': (c_int, [c_void_p, c_void_p, c_int, ctypes.c_float, ctypes.c_float, c_void_p,
                                           c_void_p, c_void_p, c_void_p]),
    'deva_b200_sam_nms_workspace_bytes': (c_size_t, [c_int]),
    'deva_b200_sam_nms': (c_int, [c_void_p, c_void_p, c_int, ctypes.c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    'deva_b200_sam_mask_write': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                         ctypes.c_float, c_void_p, c_void_p]),
}
EXPORTS = tuple(_SIGNATURES.keys())


def lib():
    """Load (once) and return the shared library; raises if it is missing or mismatched."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f'deva_b200: CUDA library not built: {LIB_PATH} (run __graft_entry__.build() or '
                               f'`make -C {os.path.dirname(LIB_PATH)}`); there is no CPU fallback')
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        if handle.deva_b200_abi_version() != ABI_VERSION:
            raise RuntimeError('deva_b200: ABI version mismatch between deva/_native.py and libdeva_b200.so')
        _lib = handle
    return _lib


def _check(rc: int, what: str):
    if rc != 0:
        msg = lib().deva_b200_last_error()
        raise RuntimeError(f'deva_b200.{what} failed ({rc}): {msg.decode() if msg else "?"}')


def _ptr(t):
    return None if t is None else c_void_p(t.data_ptr())


def _stream():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def launch_count() -> int:
    return int(lib().deva_b200_launch_count())


def require_device():
    if not torch.cuda.is_available():
        raise RuntimeError('deva_b200: no CUDA device; the sm_90a kernels have no CPU fallback')
    _check(lib().deva_b200_device_check(), 'device_check')


def _f32(t):
    assert t.dtype == torch.float32 and t.is_cuda, (t.dtype, t.device)
    return t


# ------------------------------------------------------------------------------------------ wrappers
def pack_query(qk, qe, stride_c, stride_q, ck, q, q_hi, q_lo, bsq):
    _check(lib().deva_b200_pack_query(_ptr(_f32(qk)), _ptr(_f32(qe)), stride_c, stride_q, ck, q, _ptr(q_hi),
                                      _ptr(q_lo), _ptr(bsq), _stream()), 'pack_query')


def pack_keys(key, selection, stride_c, stride_t, shrinkage, ck, n, k_hi, k_lo, neg_s, raw_key, raw_sel, raw_shr):
    _check(lib().deva_b200_pack_keys(_ptr(_f32(key)), _ptr(selection), stride_c, stride_t, _ptr(_f32(shrinkage)), ck,
                                     n, _ptr(k_hi), _ptr(k_lo), _ptr(neg_s), _ptr(raw_key), _ptr(raw_sel),
                                     _ptr(raw_shr), _stream()), 'pack_keys')


def append_values(src, ld_src, dst, ld_dst, rows, n):
    _check(lib().deva_b200_append_values(_ptr(_f32(src)), ld_src, _ptr(dst), ld_dst, rows, n, _stream()),
           'append_values')


def simtopk_workspace_bytes(q):
    return int(lib().deva_b200_simtopk_workspace_bytes(q))


def sim_topk(k_hi, k_lo, neg_s, n_window, n_lead, q_hi, q_lo, bsq, q, ck, top_k, workspace, out_idx, out_w,
             affinity, ld_affinity, use_cnt, life_cnt, n_long, count_long, count_work, out_sim=None, prev_idx=None,
             thr_ws=None):
    _check(lib().deva_b200_sim_topk(_ptr(k_hi), _ptr(k_lo), _ptr(neg_s), n_window, n_lead, _ptr(q_hi), _ptr(q_lo),
                                    _ptr(bsq), q, ck, top_k, _ptr(workspace), _ptr(out_idx), _ptr(out_w),
                                    _ptr(affinity), ld_affinity, _ptr(use_cnt), _ptr(life_cnt), n_long,
                                    int(count_long), int(count_work), _ptr(out_sim), _ptr(prev_idx), _ptr(thr_ws),
                                    _stream()), 'sim_topk')


def merge_lists(part_val, part_idx, n_lists, top_k, q, q_pitch, out_idx, out_w, out_sim=None):
    _check(lib().deva_b200_merge_lists(_ptr(part_val), _ptr(part_idx), n_lists, top_k, q, q_pitch, _ptr(out_idx),
                                       _ptr(out_w), _ptr(out_sim), _stream()), 'merge_lists')


def list_pitch(top_k: int) -> int:
    """Row pitch of the top-k lists of a read at ``top_k``: LIST_PITCH up to it, else top_k rounded up to 32."""
    return max(LIST_PITCH, (top_k + 31) // 32 * 32)


def sim_topk_wide_workspace_bytes(q, n_window):
    return int(lib().deva_b200_sim_topk_wide_workspace_bytes(q, n_window))


def sim_topk_wide(k_hi, k_lo, neg_s, n_window, n_lead, q_hi, q_lo, bsq, q, ck, top_k, workspace, out_idx, out_w,
                  ld_list, affinity, ld_affinity, use_cnt, life_cnt, n_long, count_long, count_work, out_sim=None):
    """The read at any top_k: out_idx/out_w (out_sim) [q, ld_list], selected slots in ascending slot order."""
    _check(lib().deva_b200_sim_topk_wide(_ptr(k_hi), _ptr(k_lo), _ptr(neg_s), n_window, n_lead, _ptr(q_hi),
                                         _ptr(q_lo), _ptr(bsq), q, ck, top_k, _ptr(workspace), _ptr(out_idx),
                                         _ptr(out_w), ld_list, _ptr(affinity), ld_affinity, _ptr(use_cnt),
                                         _ptr(life_cnt), n_long, int(count_long), int(count_work), _ptr(out_sim),
                                         _stream()), 'sim_topk_wide')


def merge_lists_wide(part_val, part_idx, n_lists, ld_list, top_k, q, q_pitch, out_idx, out_w, out_sim=None):
    """part_val/part_idx [n_lists, ld_list, q_pitch] -> [q, ld_list] lists, the selected entries in input order."""
    _check(lib().deva_b200_merge_lists_wide(_ptr(part_val), _ptr(part_idx), n_lists, ld_list, top_k, q, q_pitch,
                                            _ptr(out_idx), _ptr(out_w), _ptr(out_sim), _stream()), 'merge_lists_wide')


def sim_dense_softmax(k_hi, k_lo, neg_s, shrinkage, n_window, n_lead, q_hi, q_lo, bsq, q, ck, sim_ws, ld_sim,
                      affinity, ld_affinity, shr_out):
    _check(lib().deva_b200_sim_dense_softmax(_ptr(k_hi), _ptr(k_lo), _ptr(neg_s), _ptr(shrinkage), n_window, n_lead,
                                             _ptr(q_hi), _ptr(q_lo), _ptr(bsq), q, ck, _ptr(sim_ws), ld_sim,
                                             _ptr(affinity), ld_affinity, _ptr(shr_out), _stream()),
           'sim_dense_softmax')


def readout(values, values_ld, values_rows, val_row, out_row, rows_per_group, affinity, ld_affinity, n_window, q,
            out, ld_out, out_tok=None):
    n = len(val_row)
    assert n == len(out_row)
    arr_v = (c_int32 * n)(*val_row)
    arr_o = (c_int32 * n)(*out_row)
    _check(lib().deva_b200_readout(_ptr(values), values_ld, values_rows, arr_v, arr_o, n, rows_per_group,
                                   _ptr(affinity), ld_affinity, n_window, q, _ptr(out), ld_out, _ptr(out_tok),
                                   _stream()), 'readout')


def readout_sparse_workspace_bytes(q, n_window):
    return int(lib().deva_b200_readout_sparse_workspace_bytes(q, n_window))


def readout_sparse(values, values_ld, values_rows, val_row, out_row, rows_per_group, idx, w, top_k, n_window, q,
                   workspace, out, ld_out, out_tok=None):
    n = len(val_row)
    arr_v = (c_int32 * n)(*val_row)
    arr_o = (c_int32 * n)(*out_row)
    _check(lib().deva_b200_readout_sparse(_ptr(values), values_ld, values_rows, arr_v, arr_o, n, rows_per_group,
                                          _ptr(idx), _ptr(w), top_k, n_window, q, _ptr(workspace), _ptr(out), ld_out,
                                          _ptr(out_tok), _stream()), 'readout_sparse')


def readout_sparse_wide_workspace_bytes(q, n_window, ld_list):
    return int(lib().deva_b200_readout_sparse_wide_workspace_bytes(q, n_window, ld_list))


def readout_sparse_wide(values, values_ld, values_rows, val_row, out_row, rows_per_group, idx, w, ld_list, top_k,
                        n_window, q, workspace, out, ld_out, out_tok=None):
    n = len(val_row)
    arr_v = (c_int32 * n)(*val_row)
    arr_o = (c_int32 * n)(*out_row)
    _check(lib().deva_b200_readout_sparse_wide(_ptr(values), values_ld, values_rows, arr_v, arr_o, n, rows_per_group,
                                               _ptr(idx), _ptr(w), ld_list, top_k, n_window, q, _ptr(workspace),
                                               _ptr(out), ld_out, _ptr(out_tok), _stream()), 'readout_sparse_wide')


def readout_sparse_scatter_wide(values, values_ld, values_rows, val_row, out_row, owner, rows_per_group, idx, w,
                                ld_list, top_k, n_window, q, workspace, rank_dst_ptrs, ld_out):
    n = len(val_row)
    arr_v, arr_o, arr_w = (c_int32 * n)(*val_row), (c_int32 * n)(*out_row), (c_int32 * n)(*owner)
    ptrs = (c_void_p * len(rank_dst_ptrs))(*rank_dst_ptrs)
    _check(lib().deva_b200_readout_sparse_scatter_wide(_ptr(values), values_ld, values_rows, arr_v, arr_o, arr_w, n,
                                                       rows_per_group, _ptr(idx), _ptr(w), ld_list, top_k, n_window, q,
                                                       _ptr(workspace), ptrs, len(rank_dst_ptrs), ld_out, _stream()),
           'readout_sparse_scatter_wide')


def readout_sparse_scatter(values, values_ld, values_rows, val_row, out_row, owner, rows_per_group, idx, w, top_k,
                           n_window, q, workspace, rank_dst_ptrs, ld_out):
    """rank_dst_ptrs: device addresses (ints) of every rank's fp32 [objects_owned * rows_per_group, q] buffer."""
    n = len(val_row)
    arr_v, arr_o, arr_w = (c_int32 * n)(*val_row), (c_int32 * n)(*out_row), (c_int32 * n)(*owner)
    ptrs = (c_void_p * len(rank_dst_ptrs))(*rank_dst_ptrs)
    _check(lib().deva_b200_readout_sparse_scatter(_ptr(values), values_ld, values_rows, arr_v, arr_o, arr_w, n,
                                                  rows_per_group, _ptr(idx), _ptr(w), top_k, n_window, q,
                                                  _ptr(workspace), ptrs, len(rank_dst_ptrs), ld_out, _stream()),
           'readout_sparse_scatter')


def peer_alloc(device: int, nbytes: int):
    """-> (device address, 64-byte CUDA IPC handle) of a zeroed cudaMalloc'ed buffer on ``device``."""
    ptr, handle = c_void_p(), ctypes.create_string_buffer(64)
    _check(lib().deva_b200_peer_alloc(device, nbytes, ctypes.byref(ptr), handle), 'peer_alloc')
    return int(ptr.value), handle.raw


def peer_open(device: int, handle: bytes) -> int:
    ptr = c_void_p()
    _check(lib().deva_b200_peer_open(device, handle, ctypes.byref(ptr)), 'peer_open')
    return int(ptr.value)


def peer_close(device: int, ptr: int):
    _check(lib().deva_b200_peer_close(device, c_void_p(ptr)), 'peer_close')


def peer_free(device: int, ptr: int):
    _check(lib().deva_b200_peer_free(device, c_void_p(ptr)), 'peer_free')


def gather_rows(dst, src, idx, n, row_bytes):
    _check(lib().deva_b200_gather_rows(_ptr(dst), _ptr(src), _ptr(idx), n, row_bytes, _stream()), 'gather_rows')


def gather_f32(dst, src, idx, n):
    _check(lib().deva_b200_gather_f32(_ptr(dst), _ptr(src), _ptr(idx), n, _stream()), 'gather_f32')


def gather_cols_f16(dst, ld_dst, src, ld_src, idx, rows, n):
    _check(lib().deva_b200_gather_cols_f16(_ptr(dst), ld_dst, _ptr(src), ld_src, _ptr(idx), rows, n, _stream()),
           'gather_cols_f16')


def usage(out, use_cnt, life_cnt, n):
    _check(lib().deva_b200_usage(_ptr(out), _ptr(use_cnt), _ptr(life_cnt), n, _stream()), 'usage')


# ------------------------------------------------------------------------------------------ network path
def _p(t):
    return None if t is None else t.data_ptr()


def conv2d(x, batch, h, w, cin_pad, w_packed, kh, stride, cout, cout_pad, nt, th, tw, bias, x2=None, x_lo=None, res=None,
           res_lo=None, res_broadcast=False, rank1_w=None, rank1_x=None, out_raw=None, out_relu=None, out_f32=None,
           out_raw_lo=None, out_relu_lo=None, head_w=None, head_out=None, head_n=0, gate_h=None, gate_out=None,
           split_mode=0, ksplit=0, x_lo8=None, w8_packed=None, acc_scale=0.0, out_relu_lo8=None, out_pool4=None):
    d = ConvDesc(_p(x), _p(x2), _p(x_lo), split_mode, batch, h, w, cin_pad, _p(w_packed), kh, kh, stride, cout, cout_pad, nt, th, tw,
                 _p(bias), _p(res), _p(res_lo), int(res_broadcast), _p(rank1_w), _p(rank1_x), _p(out_raw), _p(out_relu),
                 _p(out_f32), _p(out_raw_lo), _p(out_relu_lo), _p(head_w), _p(head_out), head_n, _p(gate_h), _p(gate_out), _p(x_lo8), _p(w8_packed), acc_scale,
                 _p(out_relu_lo8), ksplit, _p(out_pool4))
    _check(lib().deva_b200_conv2d(ctypes.byref(d), _stream()), 'conv2d')


def stem_im2col(src, dst, b, c, h, w, k_pad, dst_lo=None):
    _check(lib().deva_b200_stem_im2col(_ptr(_f32(src)), _ptr(dst), _ptr(dst_lo), b, c, h, w, k_pad, _stream()),
           'stem_im2col')


def nchw_to_nhwc(src, dst, b, c, h, w, c_pad):
    _check(lib().deva_b200_nchw_to_nhwc(_ptr(src), _ptr(dst), b, c, h, w, c_pad, _stream()), 'nchw_to_nhwc')


def maxpool(x, y, b, h, w, c, x_lo=None, y_lo=None):
    _check(lib().deva_b200_maxpool(_ptr(x), _ptr(x_lo), _ptr(y), _ptr(y_lo), b, h, w, c, _stream()), 'maxpool')


def area_down(x, y, b, h, w, c, r):
    _check(lib().deva_b200_area_down(_ptr(x), _ptr(y), b, h, w, c, r, _stream()), 'area_down')


def area_down_plane(x, y, b, h, w, r):
    _check(lib().deva_b200_area_down_plane(_ptr(x), _ptr(y), b, h, w, r, _stream()), 'area_down_plane')


def up2_add_split(g, g_lo, skip, raw, raw_lo, relu, b, h, w, c, *, skip_lo, relu_lo8=None):
    _check(lib().deva_b200_up2_add_split(_ptr(g), _ptr(g_lo), _ptr(skip), _ptr(skip_lo), _ptr(raw), _ptr(raw_lo),
                                         _ptr(relu), _ptr(relu_lo8), b, h, w, c, _stream()), 'up2_add_split')


def cbam_split(x, x_lo, w1, b1, w2, b2, ws, bs, scratch, raw, raw_lo, relu, b, h, w, c, r):
    _check(lib().deva_b200_cbam_split(_ptr(x), _ptr(x_lo), _ptr(w1), _ptr(b1), _ptr(w2), _ptr(b2), _ptr(ws), _ptr(bs),
                                      _ptr(scratch), _ptr(raw), _ptr(raw_lo), _ptr(relu), b, h, w, c, r, _stream()),
           'cbam_split')


def sum_parts(parts, n_parts, part_stride, n, res=None, res_lo=None, raw=None, raw_lo=None, relu=None, relu_lo=None):
    _check(lib().deva_b200_sum_parts(_ptr(parts), n_parts, part_stride, _ptr(res), _ptr(res_lo), _ptr(raw), _ptr(raw_lo),
                                     _ptr(relu), _ptr(relu_lo), n, _stream()), 'sum_parts')


def key_tail(y, ld, q, ck, key, shrinkage, selection, n_parts=1, part_stride=0):
    _check(lib().deva_b200_key_tail(_ptr(y), ld, q, ck, n_parts, part_stride, _ptr(key), _ptr(shrinkage), _ptr(selection),
                                    _stream()), 'key_tail')


def output_tail(logits, agg, prob, logits_out, k, h, w):
    _check(lib().deva_b200_output_tail(_ptr(logits), _ptr(agg), _ptr(prob), _ptr(logits_out), k, h, w, _stream()),
           'output_tail')


def ingest_rgb8(src, dst, h, w, mean, std):
    m = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s = (ctypes.c_float * 3)(*[float(v) for v in std])
    _check(lib().deva_b200_ingest_rgb8(_ptr(src), _ptr(dst), h, w, m, s, _stream()), 'ingest_rgb8')


def ingest_rgb8_resize(src, h, w, out_h, out_w, x_idx, x_w, y_idx, y_w, scratch, dst, flip, mean, std):
    m = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s = (ctypes.c_float * 3)(*[float(v) for v in std])
    _check(lib().deva_b200_ingest_rgb8_resize(_ptr(src), h, w, out_h, out_w, _ptr(x_idx), _ptr(_f32(x_w)), x_w.shape[1],
                                              _ptr(y_idx), _ptr(_f32(y_w)), y_w.shape[1], _ptr(_f32(scratch)),
                                              _ptr(_f32(dst)), int(flip), m, s, _stream()), 'ingest_rgb8_resize')


def mask_nearest(src, h, w, out_h, out_w, x_idx, y_idx, flip, dst):
    _check(lib().deva_b200_mask_nearest(_ptr(src), h, w, out_h, out_w, _ptr(x_idx), _ptr(y_idx), int(flip), _ptr(dst),
                                        _stream()), 'mask_nearest')


def mask_nearest_ids(src, channels, h, w, out_h, out_w, x_idx, y_idx, flip, dst):
    _check(lib().deva_b200_mask_nearest_ids(_ptr(src), channels, h, w, out_h, out_w, _ptr(x_idx), _ptr(y_idx), int(flip),
                                            _ptr(dst), _stream()), 'mask_nearest_ids')


def pil_resample_u8(src, k, h, w, out_h, out_w, x_bounds, x_coef, y_bounds, y_coef, scratch, dst):
    _check(lib().deva_b200_pil_resample_u8(_ptr(src), k, h, w, out_h, out_w, _p(x_bounds), _p(x_coef),
                                           0 if x_coef is None else x_coef.shape[1], _p(y_bounds), _p(y_coef),
                                           0 if y_coef is None else y_coef.shape[1], _p(scratch), _ptr(_f32(dst)),
                                           _stream()), 'pil_resample_u8')


def prob_to_ids(prob, c, h, w, out_h, out_w, flip, lut, out_u8, out_i64):
    _check(lib().deva_b200_prob_to_ids(_ptr(prob), c, h, w, out_h, out_w, int(flip), _p(lut), _p(out_u8), _p(out_i64),
                                       _stream()), 'prob_to_ids')


def prob_to_segments(prob, c, h, w, out_h, out_w, lut, rgb, frame, out_u8, out_rgb, out_overlay, counts, boxes):
    _check(lib().deva_b200_prob_to_segments(_ptr(prob), c, h, w, out_h, out_w, _ptr(lut), _p(rgb), _p(frame), _p(out_u8),
                                            _p(out_rgb), _p(out_overlay), _p(counts), _p(boxes), _stream()),
           'prob_to_segments')


def prob_to_scores(prob, c, h, w, out_h, out_w, flip, scores, total):
    _check(lib().deva_b200_prob_to_scores(_ptr(prob), c, h, w, out_h, out_w, int(bool(flip)), _p(scores), _p(total),
                                          _stream()), 'prob_to_scores')


def scores_to_ids(total, c, h, w, lut, out_u8, out_i64):
    _check(lib().deva_b200_scores_to_ids(_p(total), c, h, w, _p(lut), _p(out_u8), _p(out_i64), _stream()),
           'scores_to_ids')


def pano_joint_hist(gt, pred, gt_ids, pred_ids, hist):
    """gt, pred: uint8 [h, w, 3] RGB id frames; gt_ids, pred_ids: sorted int32 tables; hist: int32 [n_gt + 1, n_pred + 1]
    (a view of a larger buffer is fine when it is contiguous)."""
    h, w = gt.shape[:2]
    assert gt.shape == pred.shape == (h, w, 3) and gt.dtype == pred.dtype == torch.uint8 and gt.is_contiguous() and \
        pred.is_contiguous(), (gt.shape, pred.shape)
    assert gt_ids.dtype == pred_ids.dtype == hist.dtype == torch.int32 and hist.is_contiguous()
    assert hist.shape == (gt_ids.numel() + 1, pred_ids.numel() + 1), hist.shape
    _check(lib().deva_b200_pano_joint_hist(_ptr(gt), _ptr(pred), h, w, _ptr(gt_ids), gt_ids.numel(), _ptr(pred_ids),
                                           pred_ids.numel(), _ptr(hist), _stream()), 'pano_joint_hist')


def pano_remap(pred, ids, slot, out_ids, out, counts, unknown):
    """pred, out: uint8 [h, w, 3]; ids: sorted int32 table; slot: int32 [len(ids) + 1]; out_ids, counts: int32 [n_out];
    unknown: int32 [1]."""
    h, w = pred.shape[:2]
    assert pred.shape == out.shape == (h, w, 3) and pred.dtype == out.dtype == torch.uint8
    assert pred.is_contiguous() and out.is_contiguous()
    assert ids.dtype == slot.dtype == out_ids.dtype == counts.dtype == unknown.dtype == torch.int32
    assert slot.numel() == ids.numel() + 1 and counts.numel() == out_ids.numel()
    _check(lib().deva_b200_pano_remap(_ptr(pred), h, w, _ptr(ids), ids.numel(), _ptr(slot), _ptr(out_ids),
                                      out_ids.numel(), _ptr(out), _ptr(counts), _ptr(unknown), _stream()), 'pano_remap')


def _label_frame(frame):
    """-> (h, w, channels) of a uint8 [h, w] or [h, w, 1 | 3 | 4] frame."""
    assert frame.dtype == torch.uint8 and frame.is_contiguous() and frame.dim() in (2, 3), (frame.dtype, frame.shape)
    return frame.shape[0], frame.shape[1], 1 if frame.dim() == 2 else frame.shape[2]


def label_areas(frame, labels, counts, state):
    """frame: uint8 [h, w] or [h, w, 3 | 4]; labels, counts: int32 [capacity]; state: int32 [2].  Enqueues the count; read
    the result with ``label_areas_result``."""
    h, w, c = _label_frame(frame)
    assert labels.dtype == counts.dtype == state.dtype == torch.int32 and labels.numel() == counts.numel()
    assert labels.is_contiguous() and counts.is_contiguous() and state.numel() == 2 and state.is_contiguous()
    _check(lib().deva_b200_label_areas(_ptr(frame), h, w, c, labels.numel(), _ptr(labels), _ptr(counts), _ptr(state),
                                       _stream()), 'label_areas')


def label_areas_result(labels, counts, state):
    """Host arrays of a completed label_areas call -> (labels, counts) [n]; raises when the frame had more distinct
    labels than the table's capacity."""
    n = int(state[0])
    if n < 0:
        raise RuntimeError(f'deva_b200.label_areas: the frame has more than {len(labels)} distinct labels (the table '
                           f'capacity)')
    return labels[:n], counts[:n]


def label_to_index(frame, labels, index, out):
    """frame: uint8 [h, w] or [h, w, 3 | 4]; labels: sorted int32 [n]; index: int32 [n]; out: uint8 [h, w]."""
    h, w, c = _label_frame(frame)
    assert labels.dtype == index.dtype == torch.int32 and labels.numel() == index.numel()
    assert out.dtype == torch.uint8 and out.shape == (h, w) and out.is_contiguous(), (out.dtype, out.shape)
    _check(lib().deva_b200_label_to_index(_ptr(frame), h, w, c, _ptr(labels), _ptr(index), labels.numel(), _ptr(out),
                                          _stream()), 'label_to_index')


def _mask_stack(masks):
    """uint8 view [n, h, w] of a contiguous bool / uint8 CUDA mask stack (no copy)."""
    assert masks.is_cuda and masks.dim() == 3 and masks.is_contiguous(), (masks.device, masks.shape)
    if masks.dtype == torch.bool:
        masks = masks.view(torch.uint8)
    if masks.dtype != torch.uint8:
        raise TypeError(f'deva_b200: mask stacks are bool or uint8, not {masks.dtype}')
    return masks


def _i32(t, n):
    assert t.dtype == torch.int32 and t.is_cuda and t.is_contiguous() and t.numel() == n, (t.dtype, t.shape, n)
    return t


def mask_stats(masks, out_h, out_w, area=None, covered=None):
    """masks bool / uint8 [n, h, w] -> area float32 [n] (deterministic fp32 sums of the resized values) and / or covered
    int32 [n] (resized values > 0.5), written into the given tensors."""
    m = _mask_stack(masks)
    n, h, w = m.shape
    if area is not None:
        assert _f32(area).numel() == n and area.is_contiguous()
    if covered is not None:
        _i32(covered, n)
    ws = torch.empty(int(lib().deva_b200_mask_stats_workspace_bytes(n, out_h, out_w)), dtype=torch.uint8,
                     device=m.device)
    _check(lib().deva_b200_mask_stats(_ptr(m), n, h, w, out_h, out_w, _ptr(ws), _ptr(area), _ptr(covered), _stream()),
           'mask_stats')


def mask_scored_argmax(masks, out_h, out_w, score, kept_only, slot, won, kept):
    """slot int32 [out_h, out_w]; won / kept int32 [n + 1]; score float32 [n] (see include/deva_b200.h)."""
    m = _mask_stack(masks)
    n, h, w = m.shape
    assert _f32(score).numel() == n and score.is_contiguous()
    _i32(slot, out_h * out_w), _i32(won, n + 1), _i32(kept, n + 1)
    _check(lib().deva_b200_mask_scored_argmax(_ptr(m), n, h, w, out_h, out_w, _ptr(score), int(bool(kept_only)),
                                              _ptr(slot), _ptr(won), _ptr(kept), _stream()), 'mask_scored_argmax')


def mask_last_cover(masks, out_h, out_w, order, slot, covered):
    """order int32 [n] (paint order); slot int32 [out_h, out_w]; covered int32 [n] (see include/deva_b200.h)."""
    m = _mask_stack(masks)
    n, h, w = m.shape
    _i32(order, n), _i32(slot, out_h * out_w), _i32(covered, n)
    _check(lib().deva_b200_mask_last_cover(_ptr(m), n, h, w, out_h, out_w, _ptr(order), _ptr(slot), _ptr(covered),
                                           _stream()), 'mask_last_cover')


def png_bound(h, w, channels, bits) -> int:
    return int(lib().deva_b200_png_bound(h, w, channels, bits))


def png_workspace_bytes(h) -> int:
    return int(lib().deva_b200_png_workspace_bytes(h))


def png_encode(img, bits, workspace, out, out_len):
    """img uint8 [h, w] or [h, w, 3]; out: png_bound bytes, 4-byte aligned; out_len int64 [1]; workspace:
    png_workspace_bytes, 8-byte aligned (see include/deva_b200.h)."""
    assert img.dtype == torch.uint8 and img.is_cuda and img.is_contiguous() and img.dim() in (2, 3), (img.dtype,
                                                                                                      img.shape)
    h, w = img.shape[:2]
    channels = 1 if img.dim() == 2 else img.shape[2]
    assert out.numel() * out.element_size() >= png_bound(h, w, channels, bits) and out_len.dtype == torch.int64
    assert workspace.numel() * workspace.element_size() >= png_workspace_bytes(h)
    _check(lib().deva_b200_png_encode(_ptr(img), h, w, channels, bits, _ptr(workspace), _ptr(out), _ptr(out_len),
                                      _stream()), 'png_encode')


def jpeg_bound(h, w) -> int:
    return int(lib().deva_b200_jpeg_bound(h, w))


def jpeg_workspace_bytes(h, w) -> int:
    return int(lib().deva_b200_jpeg_workspace_bytes(h, w))


def jpeg_encode(img, tables: bytes, workspace, out, out_len):
    """img uint8 [h, w, 3]; tables: 128 bytes (luma then chroma quantisation, zigzag); out: jpeg_bound bytes; out_len
    int64 [1]; workspace: jpeg_workspace_bytes, 16-byte aligned (see include/deva_b200.h)."""
    assert img.dtype == torch.uint8 and img.is_cuda and img.is_contiguous() and img.dim() == 3 and img.shape[2] == 3, \
        (img.dtype, img.shape)
    h, w = img.shape[:2]
    assert len(tables) == 128 and out_len.dtype == torch.int64
    assert out.numel() * out.element_size() >= jpeg_bound(h, w)
    assert workspace.numel() * workspace.element_size() >= jpeg_workspace_bytes(h, w)
    _check(lib().deva_b200_jpeg_encode(_ptr(img), h, w, bytes(tables), _ptr(workspace), _ptr(out), _ptr(out_len),
                                       _stream()), 'jpeg_encode')


def rle_bound(h, w, n) -> int:
    return int(lib().deva_b200_rle_bound(h, w, n))


def rle_workspace_bytes(h, w, n) -> int:
    return int(lib().deva_b200_rle_workspace_bytes(h, w, n))


def rle_encode(ids, seg_ids, workspace, out, offsets):
    """ids int64 [h, w]; seg_ids int64 [n]; out: rle_bound bytes; offsets int64 [n + 1]; workspace:
    rle_workspace_bytes, 16-byte aligned (see include/deva_b200.h)."""
    assert ids.dtype == torch.int64 and ids.is_cuda and ids.is_contiguous() and ids.dim() == 2, (ids.dtype, ids.shape)
    assert seg_ids.dtype == torch.int64 and seg_ids.is_cuda and seg_ids.is_contiguous() and seg_ids.dim() == 1
    h, w = ids.shape
    n = seg_ids.numel()
    assert offsets.dtype == torch.int64 and offsets.is_contiguous() and offsets.numel() == n + 1
    assert out.numel() * out.element_size() >= rle_bound(h, w, n)
    assert workspace.numel() * workspace.element_size() >= rle_workspace_bytes(h, w, n)
    _check(lib().deva_b200_rle_encode(_ptr(ids), h, w, _ptr(seg_ids), n, _ptr(workspace), _ptr(out), _ptr(offsets),
                                      _stream()), 'rle_encode')


PNG_DESC_FIELDS = 8


def png_decode_workspace_bytes(h, w, colour_type, bits) -> int:
    return int(lib().deva_b200_png_decode_workspace_bytes(h, w, colour_type, bits))


def png_decode(streams, desc, out, workspace, status):
    """streams uint8: the files' zlib streams; desc int64 [n, 8]; out uint8: the arrays at their offsets; workspace
    uint8: the filtered streams at their offsets; status int32 [n]; all on the device (see include/deva_b200.h)."""
    n = desc.shape[0]
    assert desc.dtype == torch.int64 and desc.is_cuda and desc.is_contiguous() and desc.shape == (n, PNG_DESC_FIELDS)
    assert status.dtype == torch.int32 and status.is_cuda and status.numel() == n
    for t in (streams, out, workspace):
        assert t.dtype == torch.uint8 and t.is_cuda and t.is_contiguous()
    _check(lib().deva_b200_png_decode(_ptr(streams), _ptr(desc), n, _ptr(out), _ptr(workspace), _ptr(status),
                                      _stream()), 'png_decode')


def jpeg_decode_workspace_bytes(h, w, luma_h, luma_v, subsequences) -> int:
    return int(lib().deva_b200_jpeg_decode_workspace_bytes(h, w, luma_h, luma_v, subsequences))


def jpeg_decode(scans, desc, tables, intervals, subs, out, workspace, status):
    """scans uint8: the files' unstuffed scans; desc int64 [n, 11]; tables int32 [n, 5016]; intervals int64
    [., 6]; subs int64 [., 3]; out uint8: the arrays at their offsets; workspace uint8; status int32 [n]; all on the
    device (see include/deva_b200.h)."""
    n = desc.shape[0]
    assert desc.dtype == torch.int64 and desc.is_cuda and desc.is_contiguous() and desc.shape == (n, 11)
    assert tables.dtype == torch.int32 and tables.is_cuda and tables.shape == (n, 5016)
    assert intervals.dtype == torch.int64 and subs.dtype == torch.int64 and intervals.is_cuda and subs.is_cuda
    assert status.dtype == torch.int32 and status.is_cuda and status.numel() == n
    for t in (scans, out, workspace):
        assert t.dtype == torch.uint8 and t.is_cuda and t.is_contiguous()
    _check(lib().deva_b200_jpeg_decode(_ptr(scans), _ptr(desc), n, _ptr(tables), _ptr(intervals), intervals.shape[0],
                                       _ptr(subs), subs.shape[0], _ptr(out), _ptr(workspace), _ptr(status),
                                       _stream()), 'jpeg_decode')


def transpose_append(src, dst, ld_dst, n, c):
    _check(lib().deva_b200_transpose_append(_ptr(src), _ptr(dst), ld_dst, n, c, _stream()), 'transpose_append')


def head_gather3x3(z, out, bias, b, h, w):
    _check(lib().deva_b200_head_gather3x3(_ptr(z), _ptr(out), float(bias), b, h, w, _stream()), 'head_gather3x3')


SAM_STATS = 7  # per mask: > thr + offset, > thr - offset, > thr, x0, y0, x1, y1


def _sam_logits(logits):
    assert logits.dtype == torch.float32 and logits.is_cuda and logits.is_contiguous() and logits.dim() == 3, \
        (logits.dtype, logits.shape)
    return logits.shape


def sam_mask_stats(logits, grid, in_h, in_w, out_h, out_w, iou, iou_thresh, thr_hi, thr_lo, thr, stats):
    """logits float32 [n, lh, lw]; iou float32 [n] or None; stats int32 [n, 7] (see include/deva_b200.h)."""
    n, lh, lw = _sam_logits(logits)
    assert stats.dtype == torch.int32 and stats.is_contiguous() and stats.shape == (n, SAM_STATS)
    assert iou is None or (_f32(iou).is_contiguous() and iou.numel() == n)
    _check(lib().deva_b200_sam_mask_stats(_ptr(logits), n, lh, lw, grid, in_h, in_w, out_h, out_w, _ptr(iou),
                                          iou_thresh, thr_hi, thr_lo, thr, _ptr(stats), _stream()), 'sam_mask_stats')


def sam_mask_compact(stats, iou, iou_thresh, stability_thresh, stability, boxes, kept):
    """stats int32 [n, 7] -> stability float32 [n], boxes int64 [n, 4], kept int32 [n + 1] (count, then indices)."""
    n = stats.shape[0]
    assert stats.dtype == torch.int32 and stats.is_contiguous() and stats.shape == (n, SAM_STATS)
    assert iou is None or (_f32(iou).is_contiguous() and iou.numel() == n)
    assert _f32(stability).numel() == n and boxes.dtype == torch.int64 and boxes.shape == (n, 4)
    assert kept.dtype == torch.int32 and kept.numel() == n + 1
    _check(lib().deva_b200_sam_mask_compact(_ptr(stats), _ptr(iou), n, iou_thresh, stability_thresh, _ptr(stability),
                                            _ptr(boxes), _ptr(kept), _stream()), 'sam_mask_compact')


def sam_nms(boxes, scores, iou_thresh, keep, n_keep):
    """boxes float32 [n, 4], scores float32 [n] -> keep int64 [n] (the first n_keep[0] valid), n_keep int32 [1]."""
    n = scores.numel()
    assert _f32(boxes).is_contiguous() and boxes.shape == (n, 4) and _f32(scores).is_contiguous()
    assert keep.dtype == torch.int64 and keep.numel() >= n and n_keep.dtype == torch.int32
    ws = torch.empty(int(lib().deva_b200_sam_nms_workspace_bytes(n)), dtype=torch.uint8, device=scores.device)
    _check(lib().deva_b200_sam_nms(_ptr(boxes), _ptr(scores), n, iou_thresh, _ptr(ws), _ptr(keep), _ptr(n_keep),
                                   _stream()), 'sam_nms')


def sam_mask_write(logits, sel, grid, in_h, in_w, out_h, out_w, thr, out):
    """out bool [n, out_h, out_w]: logits[sel[m]] upsampled twice, > thr; sel int64 [n]."""
    _, lh, lw = _sam_logits(logits)
    n = sel.numel()
    assert sel.dtype == torch.int64 and sel.is_cuda and sel.is_contiguous()
    assert out.dtype == torch.bool and out.is_contiguous() and out.shape == (n, out_h, out_w)
    _check(lib().deva_b200_sam_mask_write(_ptr(logits), _ptr(sel), n, lh, lw, grid, in_h, in_w, out_h, out_w, thr,
                                          _ptr(out), _stream()), 'sam_mask_write')
