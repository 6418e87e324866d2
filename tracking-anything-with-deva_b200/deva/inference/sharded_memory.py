"""Memory read of ONE bucket whose bank is sharded along the slot axis over the ranks of a process group
(BASELINE.json configs[4]: a single long video, N slots split over 8 GPUs; SURVEY.md section 8e).

The reference has no counterpart (its long-video answer is consolidation); the math is the same top-k read
(deva/model/memory_utils.py:6-76, memory_manager.py:64-75) evaluated distributedly:

  1. every rank runs the fused similarity/top-k kernel on ITS slots -> local top-k (similarity, slot) per query;
  2. all-gather of those lists (Q x 32 x 8 B per rank - ~2 MB at 1080p; Q x pitch x 8 B for top_k > 32, pitch = top_k
     rounded up to 32) over NCCL/NVLink;
  3. every rank merges the R lists with the same kernel that merges intra-GPU splits -> identical global top-k
     set and softmax weights everywhere (a plain max/sum all-reduce would not do: the softmax is over the
     GLOBAL top-k set);
  4. every rank runs the sparse-affinity readout GEMM over the selected slots it owns -> partial readout;
  5. all-reduce (sum) of the partial readouts [K*CV, Q].

Usage counters stay with the owning rank.  Data-path collectives: one all-gather (small) + one all-reduce.

``read_scatter`` replaces steps 4-5 by ONE kernel (reduce-scatter by object, SURVEY 8e "preferred"): every rank's
readout GEMM adds its tiles, straight from the epilogue (``red.add.f32`` at system scope), into the buffer of the rank
that OWNS the object - peer memory mapped through CUDA IPC, travelling over NVLink while the next tiles are still being
multiplied.  Each rank ends up with the complete readout of its K/R objects (what an object-parallel decoder consumes);
the bulk all-reduce is gone, the only collectives left are the 2 MB all-gather of candidates (which also orders the
zeroing of the buffers before the first remote add) and a one-element fence.
"""
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist

from deva import _native as nat


def shard_bounds(n_total: int, world: int, rank: int, align: int = 8) -> Tuple[int, int]:
    """Contiguous slot range [lo, hi) of ``rank``; boundaries aligned to ``align`` slots (TMA alignment of the value
    bank) except the last."""
    per = -(-n_total // world)
    per = -(-per // align) * align
    lo = min(n_total, rank * per)
    hi = min(n_total, lo + per)
    return lo, hi


def localise(idx: torch.Tensor, w: torch.Tensor, lo: int, hi: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Global (idx, weight) lists -> this shard's lists: entries owned by other ranks get weight 0 (slot 0)."""
    mine = (idx >= lo) & (idx < hi) & (w > 0)
    return torch.where(mine, idx - lo, torch.zeros_like(idx)).contiguous(), torch.where(mine, w, torch.zeros_like(w)).contiguous()


class _RawCudaArray:
    """Lets torch wrap a raw device allocation (``__cuda_array_interface__``)."""
    def __init__(self, ptr: int, shape):
        self.__cuda_array_interface__ = {'shape': tuple(shape), 'typestr': '<f4', 'data': (ptr, False), 'version': 2}


class PeerBuffers:
    """One fp32 buffer per rank; every rank maps every other rank's buffer into ITS OWN device's address space
    (CUDA IPC handle opened under the importing device with lazy peer access: NVLink P2P)."""
    def __init__(self, shape, device, group: Optional[dist.ProcessGroup] = None):
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        rank = dist.get_rank(group) if dist.is_initialized() else 0
        nbytes = 4
        for s_ in shape:
            nbytes *= int(s_)
        self.device = device
        self._own, handle = nat.peer_alloc(device.index, nbytes)
        self.local = torch.as_tensor(_RawCudaArray(self._own, shape), device=device)
        self.ptrs = [self._own]
        self._opened: List[int] = []
        if world > 1:
            handles: List = [None] * world
            dist.all_gather_object(handles, handle, group=group)
            self.ptrs = []
            for r in range(world):
                if r == rank:
                    self.ptrs.append(self._own)
                    continue
                ptr = nat.peer_open(device.index, handles[r])
                self._opened.append(ptr)
                self.ptrs.append(ptr)
            torch.cuda.synchronize(device)
            dist.barrier(group=group)

    def close(self):
        for ptr in self._opened:
            nat.peer_close(self.device.index, ptr)
        self._opened = []
        if self._own:
            self.local = None
            nat.peer_free(self.device.index, self._own)
            self._own = 0

    def __del__(self):
        try:
            self.close()
        except Exception:  # interpreter shutdown: the driver reclaims the allocation with the context
            pass


class ShardedBankReader:
    """Holds one rank's shard (packed keys + values) and performs the distributed read."""
    def __init__(self, ck: int, cv: int, num_objects: int, n_local: int, slot_offset: int, device, top_k: int = 30,
                 group: Optional[dist.ProcessGroup] = None):
        self.ck, self.cv, self.k, self.n, self.offset, self.top_k = ck, cv, num_objects, n_local, slot_offset, top_k
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.dev = device
        self.ld = (n_local + 7) // 8 * 8 + 8
        self.k_hi = torch.zeros(max(n_local, 1), 2 * ck, dtype=torch.float16, device=device)
        self.k_lo = torch.zeros_like(self.k_hi)
        self.neg_s = torch.zeros(max(n_local, 1), device=device)
        self.values = torch.zeros(num_objects * cv, self.ld, dtype=torch.float16, device=device)
        self.use_cnt = torch.zeros(max(n_local, 1), device=device)
        self._scratch = {}

    def load(self, key: torch.Tensor, shrinkage: torch.Tensor, values: torch.Tensor) -> None:
        """key fp32 [CK, n_local], shrinkage [n_local], values fp32 [K*CV, n_local] (this rank's slots)."""
        n = self.n
        if n == 0:
            return
        raw_key = torch.empty(n, self.ck, device=self.dev)
        raw_shr = torch.empty(n, device=self.dev)
        nat.pack_keys(key.contiguous(), None, n, 1, shrinkage.contiguous(), self.ck, n, self.k_hi, self.k_lo, self.neg_s,
                      raw_key, None, raw_shr)
        nat.append_values(values.contiguous(), n, self.values, self.ld, self.k * self.cv, n)

    def _buf(self, name, shape, dtype):
        need = 1
        for s_ in shape:
            need *= s_
        cur = self._scratch.get(name)
        if cur is None or cur.numel() < need or cur.dtype != dtype:
            cur = torch.empty(max(need, 1), dtype=dtype, device=self.dev)
            self._scratch[name] = cur
        return cur[:need].view(*shape)

    def _readout_ws_bytes(self, q: int, pitch: int) -> int:
        if pitch > nat.LIST_PITCH:
            return nat.readout_sparse_wide_workspace_bytes(q, self.n, pitch)
        return nat.readout_sparse_workspace_bytes(q, self.n)

    def _global_topk(self, qk: torch.Tensor, qe: torch.Tensor, q: int):
        """Steps 1-3 of a read -> (global slot ids [q, pitch], softmax weights [q, pitch], pitch).  top_k > 32 keeps
        up to top_k local candidates per rank in lists of the wider pitch and merges them with the wide kernel."""
        wide = self.top_k > nat.LIST_PITCH
        pitch = nat.list_pitch(self.top_k)
        q_hi = self._buf('q_hi', (q, 2 * self.ck), torch.float16)
        q_lo = self._buf('q_lo', (q, 2 * self.ck), torch.float16)
        bsq = self._buf('bsq', (q, ), torch.float32)
        nat.pack_query(qk.contiguous(), qe.contiguous(), q, 1, self.ck, q, q_hi, q_lo, bsq)
        # 1. local top-k (raw similarities + local slot ids)
        l_idx = self._buf('l_idx', (q, pitch), torch.int32)
        l_w = self._buf('l_w', (q, pitch), torch.float32)
        l_sim = self._buf('l_sim', (q, pitch), torch.float32)
        k_loc = min(self.top_k, self.n)
        if k_loc > 0:
            if wide:
                ws = self._buf('ws_wide', (nat.sim_topk_wide_workspace_bytes(q, self.n), ), torch.uint8)
                nat.sim_topk_wide(self.k_hi, self.k_lo, self.neg_s, self.n, 0, q_hi, q_lo, bsq, q, self.ck, k_loc, ws,
                                  l_idx, l_w, pitch, None, 0, None, None, 0, False, False, out_sim=l_sim)
            else:
                ws = self._buf('ws', (nat.simtopk_workspace_bytes(q), ), torch.uint8)
                nat.sim_topk(self.k_hi, self.k_lo, self.neg_s, self.n, 0, q_hi, q_lo, bsq, q, self.ck, k_loc, ws, l_idx,
                             l_w, None, 0, None, None, 0, False, False, out_sim=l_sim)
            valid = torch.arange(pitch, device=self.dev).view(1, -1) < k_loc
            g_idx = torch.where(valid, l_idx + self.offset, torch.full_like(l_idx, -1))
        else:
            l_sim.fill_(float('-inf'))
            g_idx = torch.full_like(l_idx, -1)
        # 2. all-gather of the candidate lists, laid out [rank][entry][query] for the merge kernel
        mine_v = l_sim.t().contiguous()
        mine_i = g_idx.t().contiguous()
        if self.world > 1:
            all_v = torch.empty(self.world, pitch, q, dtype=torch.float32, device=self.dev)
            all_i = torch.empty(self.world, pitch, q, dtype=torch.int32, device=self.dev)
            dist.all_gather_into_tensor(all_v, mine_v, group=self.group)
            dist.all_gather_into_tensor(all_i, mine_i, group=self.group)
        else:
            all_v, all_i = mine_v.unsqueeze(0), mine_i.unsqueeze(0)
        # 3. global top-k + softmax
        g_sel = self._buf('g_sel', (q, pitch), torch.int32)
        g_w = self._buf('g_w', (q, pitch), torch.float32)
        if wide:
            nat.merge_lists_wide(all_v, all_i, self.world, pitch, self.top_k, q, q, g_sel, g_w)
        else:
            nat.merge_lists(all_v, all_i, self.world, self.top_k, q, q, g_sel, g_w)
        return g_sel, g_w, pitch

    def read(self, qk: torch.Tensor, qe: torch.Tensor, count_usage: bool = True) -> torch.Tensor:
        """qk/qe fp32 [CK, Q] (replicated on every rank) -> readout fp32 [K*CV, Q] (identical on every rank)."""
        q = qk.shape[1]
        # 1-3. global top-k + softmax (same result on every rank)
        g_sel, g_w, pitch = self._global_topk(qk, qe, q)
        # 4. partial readout over the selected slots this rank owns
        idx_loc, w_loc = localise(g_sel, g_w, self.offset, self.offset + self.n)
        if count_usage and self.n > 0:
            self.use_cnt.index_add_(0, idx_loc.reshape(-1).long(), w_loc.reshape(-1))
        out = torch.zeros(self.k * self.cv, q, dtype=torch.float32, device=self.dev)
        if self.n > 0:
            rws = self._buf('rws', (self._readout_ws_bytes(q, pitch), ), torch.uint8)
            rows = [i * self.cv for i in range(self.k)]
            for i in range(0, self.k, nat.MAX_GROUPS):
                part = rows[i:i + nat.MAX_GROUPS]
                if pitch > nat.LIST_PITCH:
                    nat.readout_sparse_wide(self.values, self.ld, self.k * self.cv, part, part, self.cv, idx_loc, w_loc,
                                            pitch, pitch, self.n, q, rws, out, q)
                else:
                    nat.readout_sparse(self.values, self.ld, self.k * self.cv, part, part, self.cv, idx_loc, w_loc, pitch,
                                       self.n, q, rws, out, q)
        # 5. sum of the partial readouts
        if self.world > 1:
            dist.all_reduce(out, op=dist.ReduceOp.SUM, group=self.group)
        return out


    # ------------------------------------------------------------------ fused readout + reduce-scatter by object
    def objects_of(self, rank: int) -> Tuple[int, int]:
        per = -(-self.k // self.world)
        return min(self.k, rank * per), min(self.k, (rank + 1) * per)

    def read_scatter(self, qk: torch.Tensor, qe: torch.Tensor, count_usage: bool = True) -> torch.Tensor:
        """qk/qe fp32 [CK, Q] (replicated) -> fp32 [K_own*CV, Q]: the COMPLETE readout of the objects this rank owns
        (``objects_of(rank)``), summed over every rank's slots inside the readout kernels' epilogues."""
        q = qk.shape[1]
        per = -(-self.k // self.world)
        peers = self._scratch.get('peers')
        if peers is None or peers.local.shape[1] != q:
            if peers is not None:  # the query count changed: release the old allocation and its IPC mappings first
                torch.cuda.synchronize(self.dev)
                peers.close()
            peers = PeerBuffers((per * self.cv, q), self.dev, self.group)
            self._scratch['peers'] = peers
        peers.local.zero_()  # ordered before every remote add of this read by the all-gather below
        g_sel, g_w, pitch = self._global_topk(qk, qe, q)
        idx_loc, w_loc = localise(g_sel, g_w, self.offset, self.offset + self.n)
        if count_usage and self.n > 0:
            self.use_cnt.index_add_(0, idx_loc.reshape(-1).long(), w_loc.reshape(-1))
        if self.n > 0:
            rws = self._buf('rws', (self._readout_ws_bytes(q, pitch), ), torch.uint8)
            objs = list(range(self.k))
            for i in range(0, self.k, nat.MAX_GROUPS):
                part = objs[i:i + nat.MAX_GROUPS]
                args = (self.values, self.ld, self.k * self.cv, [o * self.cv for o in part],
                        [(o % per) * self.cv for o in part], [o // per for o in part], self.cv, idx_loc, w_loc)
                if pitch > nat.LIST_PITCH:
                    nat.readout_sparse_scatter_wide(*args, pitch, pitch, self.n, q, rws, peers.ptrs, q)
                else:
                    nat.readout_sparse_scatter(*args, pitch, self.n, q, rws, peers.ptrs, q)
        if self.world > 1:  # every rank's adds have been issued and completed before anyone consumes its buffer
            fence = self._buf('fence', (1, ), torch.float32)
            fence.zero_()
            dist.all_reduce(fence, group=self.group)
        lo, hi = self.objects_of(self.rank)
        # Lifetime: a view of the peer buffer, valid until the NEXT read_scatter of this reader (which zeroes it and lets
        # the peers add into it again); consume it on the current stream before then, or clone it.
        return peers.local[:(hi - lo) * self.cv]
