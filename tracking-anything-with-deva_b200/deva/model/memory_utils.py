"""Functional memory-read API (names of deva/model/memory_utils.py:6-94) on the sm_90a kernels.

``get_similarity`` / ``do_softmax`` / ``readout`` are what ``consensus_associated.spatial_alignment`` and user
code call directly.  The fused production path is ``MemoryManager.match_memory``; these helpers expose
the same kernels one stage at a time with reference-shaped dense tensors (batch size 1, with selection
and shrinkage - the inference configuration).
"""
from typing import Optional

import torch

from deva import _native as nat


def get_similarity(mk: torch.Tensor, ms: torch.Tensor, qk: torch.Tensor, qe: torch.Tensor,
                   add_batch_dim: bool = False) -> torch.Tensor:
    """mk [1,CK,N...], ms [1,1,N...], qk/qe [1,CK,Q...] -> similarity [1,N,Q] fp32 (memory_utils.py:6-45)."""
    if add_batch_dim:
        mk, ms, qk, qe = mk.unsqueeze(0), ms.unsqueeze(0), qk.unsqueeze(0), qe.unsqueeze(0)
    if mk.shape[0] != 1 or ms is None or qe is None:
        raise NotImplementedError('deva_b200 get_similarity: batch 1 with shrinkage and selection only')
    ck = mk.shape[1]
    key = mk[0].reshape(ck, -1).float().contiguous()
    shr = ms[0].reshape(-1).float().contiguous()
    k = qk[0].reshape(ck, -1).float().contiguous()
    e = qe[0].reshape(ck, -1).float().contiguous()
    n, q, dev = key.shape[1], k.shape[1], key.device
    k_hi = torch.empty(n, 2 * ck, dtype=torch.float16, device=dev)
    k_lo = torch.empty_like(k_hi)
    neg_s, raw_shr = torch.empty(n, device=dev), torch.empty(n, device=dev)
    raw_key = torch.empty(n, ck, device=dev)
    nat.pack_keys(key, None, n, 1, shr, ck, n, k_hi, k_lo, neg_s, raw_key, None, raw_shr)
    q_hi = torch.empty(q, 2 * ck, dtype=torch.float16, device=dev)
    q_lo = torch.empty_like(q_hi)
    bsq = torch.empty(q, device=dev)
    nat.pack_query(k, e, q, 1, ck, q, q_hi, q_lo, bsq)
    ld = (n + 7) // 8 * 8
    sim = torch.empty(q, ld, device=dev)
    aff = torch.empty(q, ld, dtype=torch.float16, device=dev)
    nat.sim_dense_softmax(k_hi, k_lo, neg_s, None, n, 0, q_hi, q_lo, bsq, q, ck, sim, ld, aff, ld, None)
    return sim[:, :n].t().unsqueeze(0)


def do_softmax(similarity: torch.Tensor, top_k: Optional[int] = None, inplace: bool = False,
               return_usage: bool = False):
    """similarity [B,N,Q] -> affinity [B,N,Q] (memory_utils.py:48-76); dense, library ops (not the hot path)."""
    if top_k is not None:
        values, indices = torch.topk(similarity, k=top_k, dim=1)
        w = torch.softmax(values, dim=1)
        affinity = (similarity.zero_() if inplace else torch.zeros_like(similarity)).scatter_(1, indices, w)
    else:
        affinity = torch.softmax(similarity, dim=1)
    if return_usage:
        return affinity, affinity.sum(dim=2)
    return affinity


def get_affinity(mk, ms, qk, qe) -> torch.Tensor:
    return do_softmax(get_similarity(mk, ms, qk, qe))


def readout(affinity: torch.Tensor, mv: torch.Tensor) -> torch.Tensor:
    """affinity [B,N,Q], mv [B,CV,T,H,W] -> [B,CV,H,W] (memory_utils.py:87-94)."""
    b, cv, t, h, w = mv.shape
    return torch.bmm(mv.view(b, cv, t * h * w), affinity).view(b, cv, h, w)
