"""One long video over the GPUs of an NVLink box: bank-sharded memory + object-parallel decode
(BASELINE.json configs[4]; SURVEY.md section 8e "bank-sharded").

The reference has no counterpart (its single-GPU answer to long videos is consolidation); what is distributed here is
exactly its per-frame math (inference_core.py:55-113,200-290; memory_manager.py:91-276):

* every rank sees every frame and runs the (cheap, object-independent) key encoder itself;
* the memory bank of a bucket is sharded along the SLOT axis: of every memory frame's h*w tokens rank r keeps the
  contiguous run ``token_bounds(hw, R, r)`` - keys, shrinkage, usage and the values of ALL objects for those tokens -
  so every rank's shard grows, consolidates and evicts in lock-step and stays 1/R of the bank;
* a read is: local fused similarity/top-k over the shard -> all-gather of the (similarity, slot) candidate lists
  (Q x 32 x 8 B per rank) -> the same merge kernel on every rank = the identical GLOBAL top-k set and softmax weights
  -> the sparse-affinity readout GEMM over the local slots whose epilogue adds every tile straight into the fp32
  buffer of the rank that OWNS the object (``red.add`` over NVLink peer memory = fused GEMM + reduce-scatter by object);
* the decoder, the value encoder and the sensory state are object-parallel: rank r owns objects
  ``[r*per, (r+1)*per)`` of the temporary-id order; the only exchanges are the all-gather of the quarter-resolution
  logits in front of the soft-aggregation (network.py:33-40 couples the objects there) and, on memory frames, the
  all-to-all that turns per-object values into per-token-slice values for the append;
* consolidation (memory_manager.py:251-276) runs on the sharded candidates: usage all-gather -> global prototype
  choice, prototype keys by all-reduce, and the candidates' softmax with its row max / row sum all-reduced over the
  ranks (the "pre-softmax max/sum" exchange), partial prototype values summed by all-reduce.

``world == 1`` (no process group) degenerates to the plain single-GPU math through the same code, which is how the
1-GPU test-suite covers it; ``tests/test_sharded_ranks_gpu.py`` runs 2, 3 and 4 ranks as processes on one GPU against float64
and the unsharded core, ``tests/test_sharded_gpu.py`` 2 ranks over NCCL on 2 GPUs.
"""
from typing import Dict, Iterable, List, Optional, Tuple

import torch
import torch.distributed as dist

from deva import _native as nat
from deva.inference.inference_core import DEVAInferenceCore
from deva.inference.memory_bank import BucketBank
from deva.inference.memory_manager import MemoryManager
from deva.inference.sharded_memory import PeerBuffers, localise


def token_bounds(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous token run [lo, hi) of ``rank`` among the n tokens of one memory frame (sizes differ by <= 1)."""
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def object_bounds(k: int, world: int, rank: int) -> Tuple[int, int]:
    """Objects [lo, hi) (positions in temporary-id order) decoded by ``rank``: blocks of ceil(k / world)."""
    per = -(-k // world) if k else 0
    return min(k, rank * per), min(k, (rank + 1) * per)


class ShardedMemoryManager(MemoryManager):
    """``MemoryManager`` whose banks hold this rank's token slice of every memory frame; all sizes it reasons about
    (HW, work / long-term budgets, prototypes) are the LOCAL ones, so the reference's bookkeeping carries over."""
    def __init__(self, config: Dict, group: Optional[dist.ProcessGroup] = None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        super().__init__(config)
        self._peers: Optional[PeerBuffers] = None
        self.all_ids: List[int] = []  # every object of the video in temporary-id order (the sensory block holds OWN ones)

    def _read_long_term_config(self, config: Dict) -> None:
        super()._read_long_term_config(config)
        if self.num_prototypes % self.world or self.max_long_tokens % self.world:
            raise RuntimeError(f'sharded bank: num_prototypes ({self.num_prototypes}) and max_long_term_elements '
                               f'({self.max_long_tokens}) must be multiples of the {self.world} ranks')
        self.global_prototypes = self.num_prototypes
        self.num_prototypes //= self.world
        self.max_long_tokens //= self.world

    # ------------------------------------------------------------------ collectives (no-ops on one rank)
    def _all_gather(self, t: torch.Tensor) -> torch.Tensor:
        """[...] -> [world, ...]"""
        if self.world == 1:
            return t.unsqueeze(0)
        out = torch.empty((self.world, ) + tuple(t.shape), dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(out, t.contiguous(), group=self.group)
        return out

    def _all_reduce(self, t: torch.Tensor, op=dist.ReduceOp.SUM) -> torch.Tensor:
        if self.world > 1:
            dist.all_reduce(t, op=op, group=self.group)
        return t

    # ------------------------------------------------------------------ objects
    def own_ids(self) -> List[int]:
        lo, hi = object_bounds(len(self.all_ids), self.world, self.rank)
        return self.all_ids[lo:hi]

    def set_objects(self, ids: List[int], sample_key: torch.Tensor) -> None:
        """The video's object list changed (new objects / purge): re-partition the per-object sensory state."""
        ids = list(ids)
        if ids == self.all_ids:
            return
        h, w = sample_key.shape[-2:]
        dev = sample_key.device
        per_old = -(-len(self.all_ids) // self.world) if self.all_ids else 0
        known: Dict[int, torch.Tensor] = {}
        if per_old and self.world > 1:
            block = torch.zeros(per_old, self.sensory_dim, h, w, dtype=torch.float16, device=dev)
            if self._sensory_block is not None and len(self._sensory_ids):
                block[:len(self._sensory_ids)] = self._sensory_block.to(torch.float16)
            every = self._all_gather(block).flatten(0, 1)  # rank-major == old temporary-id order (padded per rank)
            for r in range(self.world):
                lo, hi = object_bounds(len(self.all_ids), self.world, r)
                for j, o in enumerate(self.all_ids[lo:hi]):
                    known[o] = every[r * per_old + j]
        elif self._sensory_block is not None:
            known = {o: self._sensory_block[i] for i, o in enumerate(self._sensory_ids)}
        self.all_ids = ids
        own = self.own_ids()
        if own:
            rows = [known[o].to(torch.float16) if o in known else
                    torch.zeros(self.sensory_dim, h, w, dtype=torch.float16, device=dev) for o in own]
            self._sensory_block = torch.stack(rows).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)  # NHWC storage
        else:
            self._sensory_block = None
        self._sensory_ids = own

    def initialize_sensory_if_needed(self, sample_key: torch.Tensor, ids: List[int]):
        self.set_objects(ids, sample_key)

    def _object_order(self) -> List[int]:
        return [o for o in self.all_ids if any(o in bank.objects for bank in self._banks.values())]

    def purge_except(self, obj_keep_idx: List[int]) -> None:
        keep = set(obj_keep_idx)
        for b in list(self._banks.keys()):
            self._banks[b].keep_objects(keep)
            if not self._banks[b].objects:
                del self._banks[b]
        if not self._banks:
            self.engaged = False
        # the sensory state follows at the next set_objects() (the core calls it with the surviving ids)

    # ------------------------------------------------------------------ reading
    def match_memory(self, query_key: torch.Tensor, selection: torch.Tensor) -> torch.Tensor:
        """query_key/selection [1,CK,h,w] (replicated) -> readout [1,K_own,CV,h,w] of the objects this rank decodes,
        an API view of fp16 NHWC storage (memory_manager.py:91-169, distributed as described in the module header)."""
        h, w = query_key.shape[-2:]
        q = h * w
        dev = query_key.device
        qk, qe = self._ck_n(query_key[0]), self._ck_n(selection[0])
        if qe.stride() != qk.stride():
            qk, qe = qk.contiguous(), qe.contiguous()
        if self.read_events is not None:
            ev0 = torch.cuda.Event(enable_timing=True)
            ev0.record()
        q_hi, q_lo, bsq = self._pack_query(qk, qe, qk.stride(0), qk.stride(1), q, 'mm_')
        order = {obj: i for i, obj in enumerate(self._object_order())}
        k_total = len(order)
        per = -(-k_total // self.world)
        # top_k > 32: every rank keeps up to top_k local candidates in lists of the wider pitch, merged by the wide kernel
        wide = self.top_k > nat.LIST_PITCH
        pitch = nat.list_pitch(self.top_k)
        if self._peers is None or tuple(self._peers.local.shape) != (per * self.CV, q):
            if self._peers is not None:
                self._peers.close()
            self._peers = PeerBuffers((per * self.CV, q), dev, self.group)
        peers = self._peers
        peers.local.zero_()  # ordered before every remote add of this read by the candidate all-gather below
        ws = self._buf('topk_ws', (nat.simtopk_workspace_bytes(q), ), torch.uint8, dev)
        l_w = self._buf('l_w', (q, pitch), torch.float32, dev)
        thr_ws = self._buf('topk_thr', (q, ), torch.float32, dev)
        l_sim = self._buf('l_sim', (q, pitch), torch.float32, dev)
        g_sel = self._buf('g_sel', (q, pitch), torch.int32, dev)
        g_w = self._buf('g_w', (q, pitch), torch.float32, dev)
        col = torch.arange(pitch, device=dev).view(1, -1)
        for bank in self._banks.values():
            w0, lead, n_window = bank.window()
            n_loc = n_window - lead
            # global slot id = rank * 2^24 + local slot: unique across ranks, only used to tell the owners apart
            stride = 1 << 24
            assert n_window < stride
            k_loc = min(self.top_k, n_loc)
            if wide:
                l_idx = self._buf('l_idx_wide', (q, pitch), torch.int32, dev)
                bank.read_key = None  # the next narrow read starts cold
            else:
                l_idx, prev = self._read_slots(bank, q, w0, lead, dev)  # the LOCAL top-k of the previous frame bounds this one's
                if bank.read_key is not None and getattr(bank, 'read_k', None) != k_loc:
                    prev = None
                bank.read_k = k_loc
            if k_loc > 0 and wide:
                wws = self._buf('topk_wide_ws', (nat.sim_topk_wide_workspace_bytes(q, n_window), ), torch.uint8, dev)
                nat.sim_topk_wide(bank.k_hi[w0:], bank.k_lo[w0:], bank.neg_s[w0:], n_window, lead, q_hi, q_lo, bsq, q,
                                  self.CK, k_loc, wws, l_idx, l_w, pitch, None, 0, None, None, 0, False, False,
                                  out_sim=l_sim)
            elif k_loc > 0:
                nat.sim_topk(bank.k_hi[w0:], bank.k_lo[w0:], bank.neg_s[w0:], n_window, lead, q_hi, q_lo, bsq, q, self.CK,
                             k_loc, ws, l_idx, l_w, None, 0, None, None, 0, False, False, out_sim=l_sim, prev_idx=prev,
                             thr_ws=thr_ws)
            if k_loc > 0:
                g_idx = torch.where(col < k_loc, l_idx + self.rank * stride, torch.full_like(l_idx, -1))
            else:
                l_sim.fill_(float('-inf'))
                g_idx = torch.full_like(l_idx, -1)
            all_v = self._all_gather(l_sim.t().contiguous())
            all_i = self._all_gather(g_idx.t().contiguous())
            if wide:
                nat.merge_lists_wide(all_v, all_i, self.world, pitch, self.top_k, q, q, g_sel, g_w)
            else:
                nat.merge_lists(all_v, all_i, self.world, self.top_k, q, q, g_sel, g_w)
            idx_loc, w_loc = localise(g_sel, g_w, self.rank * stride, self.rank * stride + n_window)
            if self.use_long_term and n_loc > 0:  # usage of MY slots under the global softmax (kv_memory_store.py:118-125)
                count_long = self.count_long_term_usage and bank.long_size > 0
                lo = bank.lo if count_long else bank.base
                phys = (idx_loc.reshape(-1).long() + w0)
                wv = torch.where(phys >= lo, w_loc.reshape(-1), torch.zeros_like(w_loc.reshape(-1)))
                bank.use_cnt.index_add_(0, phys, wv)
                bank.life_cnt[lo:bank.hi] += 1
            if n_loc > 0:
                rws_bytes = nat.readout_sparse_wide_workspace_bytes(q, n_window, pitch) if wide else \
                    nat.readout_sparse_workspace_bytes(q, n_window)
                rws = self._buf('readout_ws', (rws_bytes, ), torch.uint8, dev)
                objs = bank.objects
                for i in range(0, len(objs), nat.MAX_GROUPS):
                    part = objs[i:i + nat.MAX_GROUPS]
                    args = (bank.values[:, :, w0:], bank.cap, bank.values.shape[0] * self.CV,
                            [bank.slot_of[o] * self.CV for o in part], [(order[o] % per) * self.CV for o in part],
                            [order[o] // per for o in part], self.CV, idx_loc, w_loc)
                    if wide:
                        nat.readout_sparse_scatter_wide(*args, pitch, pitch, n_window, q, rws, peers.ptrs, q)
                    else:
                        nat.readout_sparse_scatter(*args, pitch, n_window, q, rws, peers.ptrs, q)
        if self.world > 1:  # every rank's adds are complete before anyone consumes its buffer
            fence = torch.zeros(1, device=dev)
            dist.all_reduce(fence, group=self.group)
        lo, hi = object_bounds(k_total, self.world, self.rank)
        k_own = hi - lo
        out = torch.empty(max(k_own, 1), h, w, self.CV, dtype=torch.float16, device=dev)
        if k_own:
            nat.nchw_to_nhwc(peers.local, out, k_own, self.CV, h, w, self.CV)
        if self.read_events is not None:
            ev1 = torch.cuda.Event(enable_timing=True)
            ev1.record()
            self.read_events.append((ev0, ev1))
        return out[:k_own].permute(0, 3, 1, 2).unsqueeze(0)

    # ------------------------------------------------------------------ long-term maintenance on sharded candidates
    def _long_size(self, bank: BucketBank) -> int:
        """Local sizes can drift apart after evictions (ties); every rank must take the same branch."""
        if self.world == 1:
            return bank.long_size
        return int(self._all_reduce(torch.tensor([bank.long_size], device=bank.device)).item()) // self.world

    def _evict_long(self, bank: BucketBank, max_size: int) -> None:
        """remove_obsolete_features (kv_memory_store.py:164-185) with the GLOBAL usage threshold."""
        if self.world == 1:
            return bank.evict_long(max_size)
        dev = bank.device
        n = bank.long_size
        sizes = self._all_gather(torch.tensor([n], device=dev)).view(-1)
        n_max, n_all = int(sizes.max()), int(sizes.sum())
        usage = torch.full((n_max, ), float('inf'), device=dev)
        if n:
            nat.usage(usage, bank.use_cnt[bank.lo:], bank.life_cnt[bank.lo:], n)
        every = self._all_gather(usage).view(-1)
        drop = n_all - max_size * self.world
        smallest, _ = torch.topk(every, k=drop, largest=False, sorted=True)
        keep = torch.nonzero(usage[:n] > smallest[-1]).reshape(-1).to(torch.int32) + bank.lo  # strict '>' (quirk Q5)
        kept = int(keep.numel())
        bank._compact(keep, bank.base - kept)
        bank.lo = bank.base - kept

    def consolidation(self, bank: BucketBank, c0: int, c1: int):
        """Prototype selection + potentiation over the SHARDED candidates [c0, c1) of every rank
        (memory_manager.py:251-276).  Returns this rank's slice of the global prototypes."""
        if self.world == 1:
            return super().consolidation(bank, c0, c1)
        dev = bank.device
        n_cand, p_all, p_loc = c1 - c0, self.global_prototypes, self.num_prototypes
        # 1. global top-P usage over all ranks' candidates
        n_max = int(self._all_reduce(torch.tensor([n_cand], device=dev), dist.ReduceOp.MAX).item())
        usage = torch.full((n_max, ), float('-inf'), device=dev)
        nat.usage(usage, bank.use_cnt[c0:], bank.life_cnt[c0:], n_cand)
        every = self._all_gather(usage).view(-1)
        _, top = torch.topk(every, k=p_all, dim=-1, sorted=True)
        owner, local = top // n_max, top % n_max
        mine = owner == self.rank
        # 2. prototype keys / selections: the owner contributes the row, the all-reduce delivers it to everyone
        src = torch.where(mine, local + c0, torch.full_like(local, c0)).to(torch.int32)
        proto_key = torch.empty(p_all, self.CK, dtype=torch.float32, device=dev)
        proto_sel = torch.empty(p_all, self.CK, dtype=torch.float32, device=dev)
        nat.gather_rows(proto_key, bank.raw_key, src, p_all, self.CK * 4)
        nat.gather_rows(proto_sel, bank.raw_sel, src, p_all, self.CK * 4)
        both = torch.stack([proto_key, proto_sel]) * mine.view(1, -1, 1).to(torch.float32)
        self._all_reduce(both)
        proto_key, proto_sel = both[0].contiguous(), both[1].contiguous()
        q_hi, q_lo, bsq = self._pack_query(proto_key, proto_sel, 1, self.CK, p_all, 'co_')
        # 3. similarity of every prototype to MY candidates; softmax over ALL candidates: row max and row sum are
        #    all-reduced over the ranks (memory_utils.py:66-71 evaluated distributedly)
        w0, lead, n_window = bank.window(c0, c1)
        ld = (n_window + 7) // 8 * 8
        sim = self._buf('co_sim', (p_all, ld), torch.float32, dev)
        aff = self._buf('co_aff', (p_all, ld), torch.float16, dev)
        scratch_shr = torch.empty(p_all, dtype=torch.float32, device=dev)
        nat.sim_dense_softmax(bank.k_hi[w0:], bank.k_lo[w0:], bank.neg_s[w0:], bank.raw_shr[w0:], n_window, lead,
                              q_hi, q_lo, bsq, p_all, self.CK, sim, ld, aff, ld, scratch_shr)
        s = sim[:, lead:n_window]
        m = self._all_reduce(s.max(dim=1, keepdim=True)[0], dist.ReduceOp.MAX)
        e = torch.exp(s - m)
        z = self._all_reduce(e.sum(dim=1, keepdim=True))
        pw = e / z
        aff.zero_()
        aff[:, lead:n_window] = pw.to(torch.float16)
        proto_shr = self._all_reduce((pw * bank.raw_shr[w0 + lead:w0 + n_window].view(1, -1)).sum(1))
        # 4. partial prototype values over my candidates, summed over the ranks
        live = bank.objects
        proto_val = torch.zeros(len(live) * self.CV, p_all, dtype=torch.float32, device=dev)
        for i in range(0, len(live), nat.MAX_GROUPS):
            part = live[i:i + nat.MAX_GROUPS]
            nat.readout(bank.values[:, :, w0:], bank.cap, bank.values.shape[0] * self.CV,
                        [bank.slot_of[o] * self.CV for o in part], [(i + j) * self.CV for j in range(len(part))],
                        self.CV, aff, ld, n_window, p_all, proto_val, p_all)
        self._all_reduce(proto_val)
        a, b = self.rank * p_loc, (self.rank + 1) * p_loc  # every rank stores its 1/R of the prototypes
        return proto_key[a:b].contiguous(), proto_val[:, a:b].contiguous(), proto_shr[a:b].contiguous()


class ShardedDEVAInferenceCore(DEVAInferenceCore):
    """``DEVAInferenceCore`` for ONE video driven in lock-step by every rank of ``group`` (same frames, masks and
    calls on every rank); each rank returns the full [K+1, H, W] probabilities."""
    def __init__(self, network, config: Dict, *, group: Optional[dist.ProcessGroup] = None, image_feature_store=None):
        super().__init__(network, config, image_feature_store=image_feature_store)
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.memory = ShardedMemoryManager(config, group)

    def _own(self, k: int) -> slice:
        lo, hi = object_bounds(k, self.world, self.rank)
        return slice(lo, hi)

    def _segment(self, key: torch.Tensor, selection: torch.Tensor, ms_features: Iterable[torch.Tensor],
                 update_sensory: bool = True) -> torch.Tensor:
        mem = self.memory
        if not mem.engaged:
            return super()._segment(key, selection, ms_features, update_sensory)
        eng = self.network.engine
        ids = self.object_manager.all_obj_ids
        mem.set_objects(ids, key)
        k = len(ids)
        own = self._own(k)
        k_own = own.stop - own.start
        per = -(-k // self.world)
        readout = mem.match_memory(key, selection)
        h4, w4 = key.shape[-2] * 4, key.shape[-1] * 4
        mine = torch.zeros(per, h4, w4, dtype=torch.float32, device=key.device)
        if k_own:
            sensory, logits = eng.decode(ms_features, readout, mem.get_sensory(mem.own_ids()), self.last_mask[:, own],
                                         update_sensory=update_sensory, chunk_size=self.chunk_size)
            mine[:k_own] = logits[0]
            if update_sensory:
                mem.update_sensory(sensory, mem.own_ids())
        # soft-aggregation couples the objects (network.py:33-40): gather every rank's quarter-resolution logits
        every = mem._all_gather(mine).flatten(0, 1)
        if per * self.world != k:  # ragged last rank(s): drop the padding rows
            rows = [r * per + j for r in range(self.world) for j in range(object_bounds(k, self.world, r)[1] -
                                                                          object_bounds(k, self.world, r)[0])]
            every = every[rows]
        _, prob = eng.probabilities(every.unsqueeze(0).contiguous())
        return prob[0]

    def _add_memory(self, image: torch.Tensor, ms_features: Iterable[torch.Tensor], prob: torch.Tensor,
                    key: torch.Tensor, shrinkage: torch.Tensor, selection: torch.Tensor, *,
                    is_deep_update: bool = True) -> None:
        if prob.shape[1] == 0:
            return super()._add_memory(image, ms_features, prob, key, shrinkage, selection, is_deep_update=is_deep_update)
        mem = self.memory
        ids = self.object_manager.all_obj_ids
        mem.set_objects(ids, key)
        k = len(ids)
        own = self._own(k)
        k_own = own.stop - own.start
        per = -(-k // self.world)
        h, w = key.shape[-2:]
        n = h * w
        cv = self.network.value_dim
        dev = key.device
        t0, t1 = token_bounds(n, self.world, self.rank)
        # value encoder on my objects -> fp16 token-major [K_own, n, CV]
        tok = torch.zeros(per, n, cv, dtype=torch.float16, device=dev)
        if k_own:
            value, sensory = self.network.encode_mask(image, ms_features, mem.get_sensory(mem.own_ids()), prob[:, own],
                                                      is_deep_update=is_deep_update, chunk_size=self.chunk_size)
            tok[:k_own] = value[0].permute(0, 2, 3, 1).reshape(k_own, n, cv)
            if is_deep_update:
                mem.update_sensory(sensory, mem.own_ids())
        # per-object values -> per-token-slice values of ALL objects (all-to-all; sizes differ by <= 1 token)
        if self.world > 1:
            n_max = -(-n // self.world)
            send = torch.zeros(self.world, per, n_max, cv, dtype=torch.float16, device=dev)
            for r in range(self.world):
                a, b = token_bounds(n, self.world, r)
                send[r, :, :b - a] = tok[:, a:b]
            recv = torch.empty_like(send)
            dist.all_to_all_single(recv, send, group=self.group)
            vals = recv[:, :, :t1 - t0].reshape(self.world * per, t1 - t0, cv)  # rank-major == temporary-id order (+ padding)
            if per * self.world != k:
                rows = [r * per + j for r in range(self.world) for j in range(object_bounds(k, self.world, r)[1] -
                                                                              object_bounds(k, self.world, r)[0])]
                vals = vals[rows]
            vals = vals.contiguous()
        else:
            vals = tok[:k]
        n_loc = t1 - t0
        value_loc = vals.permute(0, 2, 1).unsqueeze(-1).unsqueeze(0)  # [1, K, CV, n_loc, 1] view of token-major storage
        key_loc = mem._ck_n(key[0])[:, t0:t1].reshape(1, -1, n_loc, 1)
        shr_loc = shrinkage[0].reshape(1, n)[:, t0:t1].reshape(1, 1, n_loc, 1)
        sel_loc = mem._ck_n(selection[0])[:, t0:t1].reshape(1, -1, n_loc, 1) if selection is not None else None
        mem.add_memory(key_loc, shr_loc, value_loc, ids, selection=sel_loc)
        self.last_mem_ti = self.curr_ti
