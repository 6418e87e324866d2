"""Working / long-term / sensory memory on H100 (API of deva/inference/memory_manager.py:14-292).

Same class, method names, argument meaning and error behaviour as the reference's ``MemoryManager``;
the math runs in the sm_90a kernels behind ``deva._native``:

* ``match_memory``  = pack_query -> per bucket [sim_topk (fused similarity / top-k / softmax / usage; sim_topk_wide
  for top_k > 32) -> readout GEMM] writing straight into one [K, CV, h, w] buffer in temporary-id order;
* ``add_memory``    = O(new tokens) append into the preallocated bank (no torch.cat);
* ``compress_features`` / ``consolidation`` = the same kernels with the full-softmax variant.

There is no PyTorch fallback for any of these.
"""
from typing import Dict, List, Optional, Tuple

import torch

from deva import _native as nat
from deva.inference.kv_memory_store import KeyValueMemoryStore
from deva.inference.memory_bank import BucketBank


class MemoryManager:
    def __init__(self, config: Dict):
        nat.lib()  # fail now, not at the first frame, if the CUDA library is missing
        self.sensory_dim = config['value_dim']
        self.top_k = config['top_k']
        self.use_long_term = config['enable_long_term']
        self.count_long_term_usage = config['enable_long_term_count_usage']
        self.chunk_size = config['chunk_size']
        if self.use_long_term:
            self._read_long_term_config(config)

        self.CK = self.CV = None
        self.H = self.W = None
        self.HW = None

        self._banks: Dict[int, BucketBank] = {}
        self._next_bucket = 0
        self.work_mem = KeyValueMemoryStore(self._banks, 'work', save_selection=self.use_long_term,
                                            save_usage=self.use_long_term)
        if self.use_long_term:
            self.long_mem = KeyValueMemoryStore(self._banks, 'long', save_usage=self.count_long_term_usage)

        # sensory memory: one [K, C, h, w] block in temporary-id order + the ids it holds
        self._sensory_ids: List[int] = []
        self._sensory_block: Optional[torch.Tensor] = None
        self._scratch: Dict[str, torch.Tensor] = {}

        self.config_stale = True
        self.engaged = False
        # optional profiling hook: a list that receives one (start, end) CUDA-event pair per match_memory call
        self.read_events = None
        # 'nhwc' (the product layout): match_memory returns fp16 views of token-major storage, which the NHWC decoder
        # consumes as they are; 'nchw': fp32 [CV,h,w] in the reference's layout
        self.readout_layout = 'nhwc'
        self.fused_min_work = 16_000_000  # n_window * q above which the fused sparse-affinity readout is used
        self.work_frames_without_long_term = 16  # bank capacity (frames) when long-term memory is disabled

    def _read_long_term_config(self, config: Dict) -> None:
        self.max_mem_frames = config['max_mid_term_frames']
        self.min_mem_frames = config['min_mid_term_frames']
        self.num_prototypes = config['num_prototypes']
        self.max_long_tokens = config['max_long_term_elements']

    def update_config(self, config: Dict) -> None:
        self.config_stale = True
        self.sensory_dim = config['value_dim']
        self.top_k = config['top_k']
        assert self.use_long_term == config['enable_long_term'], 'cannot update this'
        assert self.count_long_term_usage == config['enable_long_term_count_usage'], 'cannot update this'
        if self.use_long_term:
            self._read_long_term_config(config)

    # ------------------------------------------------------------------ scratch
    def _buf(self, name: str, shape: Tuple[int, ...], dtype, device) -> torch.Tensor:
        """Grow-only scratch buffers, reused across frames (no per-frame allocation on the hot path)."""
        need = 1
        for s in shape:
            need *= s
        cur = self._scratch.get(name)
        if cur is None or cur.numel() < need or cur.dtype != dtype or cur.device != device:
            cur = torch.empty(max(need, 1), dtype=dtype, device=device)
            self._scratch[name] = cur
        return cur[:need].view(*shape)

    @staticmethod
    def _ck_n(t: torch.Tensor) -> torch.Tensor:
        """[CK, h, w] API tensor -> fp32 [CK, n] view with unit stride along one axis (no copy when possible)."""
        ck, h, w = t.shape
        if t.dtype == torch.float32:
            if t.is_contiguous():
                return t.view(ck, h * w)
            if t.stride() == (1, w * ck, ck):  # token-major storage (NHWC engine)
                return t.as_strided((ck, h * w), (1, ck), t.storage_offset())
        return t.reshape(ck, h * w).float().contiguous()

    def _pack_query(self, qk: torch.Tensor, qe: torch.Tensor, stride_c: int, stride_q: int, q: int, tag: str):
        dev = qk.device
        q_hi = self._buf(tag + 'q_hi', (q, 2 * self.CK), torch.float16, dev)
        q_lo = self._buf(tag + 'q_lo', (q, 2 * self.CK), torch.float16, dev)
        bsq = self._buf(tag + 'bsq', (q, ), torch.float32, dev)
        nat.pack_query(qk, qe, stride_c, stride_q, self.CK, q, q_hi, q_lo, bsq)
        return q_hi, q_lo, bsq

    # ------------------------------------------------------------------ reading
    def _readout(self, affinity, v) -> torch.Tensor:
        """Dense helper kept for API parity (memory_manager.py:64-75): v [C,N] or [K,C,N] times affinity [N,Q]."""
        if v.dim() == 2:
            return v.to(affinity.dtype) @ affinity
        k, c, n = v.shape
        return (v.reshape(k * c, n).to(affinity.dtype) @ affinity).view(k, c, -1)

    def match_memory(self, query_key: torch.Tensor, selection: torch.Tensor) -> Dict[int, torch.Tensor]:
        """query_key/selection [1,CK,h,w] -> {object id: readout [CV,h,w]} (memory_manager.py:91-169)."""
        assert query_key.shape[0] == 1
        h, w = query_key.shape[-2:]
        q = h * w
        dev = query_key.device
        qk = self._ck_n(query_key[0])
        qe = self._ck_n(selection[0])
        if qe.stride() != qk.stride():
            qk, qe = qk.contiguous(), qe.contiguous()
        if self.read_events is not None:
            ev0 = torch.cuda.Event(enable_timing=True)
            ev0.record()
        q_hi, q_lo, bsq = self._pack_query(qk, qe, qk.stride(0), qk.stride(1), q, 'mm_')

        order = {obj: i for i, obj in enumerate(self._object_order())}
        k_total = len(order)
        nhwc = self.readout_layout == 'nhwc'
        if nhwc:  # fp16 [K, q, CV]: per object a [CV,h,w]-shaped view of token-major storage
            out, out_tok = None, torch.empty(k_total, q, self.CV, dtype=torch.float16, device=dev)
        else:     # fp32 [K*CV, q]: the reference's layout
            out, out_tok = torch.empty(k_total * self.CV, q, dtype=torch.float32, device=dev), None
        # top_k beyond the 32-entry running lists of sim_topk: exact radix select over a dense similarity row, lists
        # at a wider pitch, no warm start
        wide = self.top_k > nat.LIST_PITCH
        pitch = nat.list_pitch(self.top_k)
        if wide:
            wgt = self._buf('topk_w', (q, pitch), torch.float32, dev)
            wide_idx = self._buf('topk_idx', (q, pitch), torch.int32, dev)
        else:
            ws = self._buf('topk_ws', (nat.simtopk_workspace_bytes(q), ), torch.uint8, dev)
            wgt = self._buf('topk_w', (q, nat.LIST_PITCH), torch.float32, dev)
            thr_ws = self._buf('topk_thr', (q, ), torch.float32, dev)
        for bank in self._banks.values():
            w0, lead, n_window = bank.window()
            count_work = self.use_long_term
            count_long = self.use_long_term and self.count_long_term_usage and bank.long_size > 0
            # large reads: affinity tiles are generated on chip by the readout kernel; small reads (where its fixed
            # costs dominate): dense fp16 affinity + plain GEMM
            fused = n_window * q >= self.fused_min_work
            aff, ldp = None, 0
            if not fused:
                ldp = (n_window + 7) // 8 * 8
                aff = self._buf('affinity', (q, ldp), torch.float16, dev)
            use = bank.use_cnt[w0:] if count_work else None
            life = bank.life_cnt[w0:] if count_work else None
            if wide:
                idx = wide_idx
                bank.read_key = None  # the next narrow read starts cold
                ws = self._buf('topk_wide_ws', (nat.sim_topk_wide_workspace_bytes(q, n_window), ), torch.uint8, dev)
                nat.sim_topk_wide(bank.k_hi[w0:], bank.k_lo[w0:], bank.neg_s[w0:], n_window, lead, q_hi, q_lo, bsq, q,
                                  self.CK, self.top_k, ws, idx, wgt, pitch, aff, ldp, use, life, bank.base - w0,
                                  count_long, count_work)
            else:
                idx, prev = self._read_slots(bank, q, w0, lead, dev)
                nat.sim_topk(bank.k_hi[w0:], bank.k_lo[w0:], bank.neg_s[w0:], n_window, lead, q_hi, q_lo, bsq, q,
                             self.CK, self.top_k, ws, idx, wgt, aff, ldp, use, life,
                             bank.base - w0, count_long, count_work, prev_idx=prev, thr_ws=thr_ws)
            objs = bank.objects
            if fused:
                rws_bytes = nat.readout_sparse_wide_workspace_bytes(q, n_window, pitch) if wide else \
                    nat.readout_sparse_workspace_bytes(q, n_window)
                rws = self._buf('readout_ws', (rws_bytes, ), torch.uint8, dev)
            for i in range(0, len(objs), nat.MAX_GROUPS):
                part = objs[i:i + nat.MAX_GROUPS]
                rows_v = [bank.slot_of[o] * self.CV for o in part]
                rows_o = [order[o] * self.CV for o in part]
                if fused and wide:
                    nat.readout_sparse_wide(bank.values[:, :, w0:], bank.cap, bank.values.shape[0] * self.CV, rows_v,
                                            rows_o, self.CV, idx, wgt, pitch, self.top_k, n_window, q, rws, out, q,
                                            out_tok)
                elif fused:
                    nat.readout_sparse(bank.values[:, :, w0:], bank.cap, bank.values.shape[0] * self.CV, rows_v, rows_o,
                                       self.CV, idx, wgt, self.top_k, n_window, q, rws, out, q, out_tok)
                else:
                    nat.readout(bank.values[:, :, w0:], bank.cap, bank.values.shape[0] * self.CV, rows_v, rows_o,
                                self.CV, aff, ldp, n_window, q, out, q, out_tok)
        if self.read_events is not None:
            ev1 = torch.cuda.Event(enable_timing=True)
            ev1.record()
            self.read_events.append((ev0, ev1))
        if nhwc:
            out = out_tok.view(k_total, h, w, self.CV).permute(0, 3, 1, 2)
        else:
            out = out.view(k_total, self.CV, h, w)
        return {obj: out[i] for obj, i in order.items()}

    def _read_slots(self, bank: BucketBank, q: int, w0: int, lead: int, dev):
        """(idx buffer of this bank's read, previous selection or None).  Temporal warm start: while the bank's slot
        numbering is unchanged (appends keep it) the slots selected for each query in the previous frame bound this
        frame's k-th best similarity from below, and the top-k kernel only inserts candidates above that bound."""
        key = (bank.numbering, w0, lead, q, self.top_k)
        if bank.read_idx is None or bank.read_idx.shape[0] != q or bank.read_idx.device != dev:
            bank.read_idx = torch.empty(q, nat.LIST_PITCH, dtype=torch.int32, device=dev)
            bank.read_key = None
        prev = bank.read_idx if bank.read_key == key else None
        bank.read_key = key
        return bank.read_idx, prev

    def _object_order(self) -> List[int]:
        """Objects in the order they entered memory == temporary-id order of the object manager."""
        return [o for b in sorted(self._banks) for o in self._banks[b].objects] if not self._sensory_ids else \
            [o for o in self._sensory_ids if any(o in bank.slot_of and o in bank.objects for bank in self._banks.values())]

    # ------------------------------------------------------------------ writing
    def add_memory(self, key: torch.Tensor, shrinkage: torch.Tensor, value: torch.Tensor, objects: List[int],
                   selection: torch.Tensor = None) -> None:
        """key [1,CK,h,w], shrinkage [1,1,h,w], value [1,K,CV,h,w], objects: ids in value order (:171-218)."""
        self.engaged = True
        if self.H is None or self.config_stale:
            self.config_stale = False
            self.H, self.W = value.shape[-2:]
            self.HW = self.H * self.W
            if self.use_long_term:
                self.max_work_tokens = self.max_mem_frames * self.HW
                self.min_work_tokens = self.min_mem_frames * self.HW
        n = key.shape[-2] * key.shape[-1]
        key = self._ck_n(key[0])
        shr = shrinkage[0].reshape(n).float().contiguous()
        self.CK = key.shape[0]
        v0 = value[0]  # [K, CV, h, w]
        self.CV = v0.shape[1]
        if v0.dtype == torch.float16 and v0.permute(0, 2, 3, 1).is_contiguous():
            value = v0.as_strided((v0.shape[0], self.CV, n), (n * self.CV, 1, self.CV), v0.storage_offset())
        else:
            value = v0.reshape(v0.shape[0], self.CV, n).float()
        sel = None
        if selection is not None and self.use_long_term:
            sel = self._ck_n(selection[0])
            if sel.stride() != key.stride():
                key, sel = key.contiguous(), sel.contiguous()

        # kv_memory_store.py:67-90: known objects extend their bucket, unknown ones open ONE new bucket
        per_bank: Dict[int, Dict[int, torch.Tensor]] = {}
        fresh: List[int] = []
        for i, obj in enumerate(objects):
            owner = [b for b, bank in self._banks.items() if obj in bank.objects]
            if owner:
                assert len(owner) == 1
                per_bank.setdefault(owner[0], {})[obj] = value[i]
            else:
                fresh.append(i)
        if fresh:
            b = self._next_bucket
            self._next_bucket += 1
            ids = [objects[i] for i in fresh]
            if self.use_long_term:
                long_cap, work_cap = self.max_long_tokens, self.max_work_tokens + n
            else:
                long_cap, work_cap = 0, self.work_frames_without_long_term * n
            self._banks[b] = BucketBank(ids, self.CK, self.CV, long_cap, work_cap, key.device)
            per_bank[b] = {objects[i]: value[i] for i in fresh}
        for b, vals in per_bank.items():
            self._banks[b].append_work(key, shr, sel, vals)

        if self.use_long_term:
            self._maintain_long_term()

    def _maintain_long_term(self) -> None:
        """Long-term clean-up after an append (memory_manager.py:207-218)."""
        for b in list(self._banks.keys()):
            bank = self._banks[b]
            if bank.work_size >= self.max_work_tokens:
                if self._long_size(bank) >= (self.max_long_tokens - self.num_prototypes):
                    if not self.count_long_term_usage:
                        raise RuntimeError('I did not count usage!')  # kv_memory_store.py:189-190
                    self._evict_long(bank, self.max_long_tokens - self.num_prototypes)
                self.compress_features(b)

    def _long_size(self, bank: BucketBank) -> int:
        return bank.long_size

    def _evict_long(self, bank: BucketBank, max_size: int) -> None:
        bank.evict_long(max_size)

    def compress_features(self, bucket_id: int) -> None:
        """Consolidate the middle of the working memory into prototypes (memory_manager.py:231-249)."""
        bank, hw = self._banks[bucket_id], self.HW
        start = hw
        end = -self.min_work_tokens + hw
        stop = bank.work_size + end if end != 0 else bank.work_size
        proto_key, proto_val, proto_shr = self.consolidation(bank, bank.base + start, bank.base + stop)
        if bank.work_size > self.min_work_tokens + hw and end != 0:  # sieve_by_range's min_size rule (:133-135)
            bank.drop_work_range(start, end)
        bank.prepend_long(proto_key, proto_shr, proto_val)

    def consolidation(self, bank: BucketBank, c0: int, c1: int):
        """Prototype selection + potentiation on candidate tokens [c0, c1) (memory_manager.py:251-276).

        Returns (prototype keys [P,CK], prototype values [len(objects)*CV, P] fp32, prototype shrinkage [P]).
        """
        dev = bank.device
        n_cand, p = c1 - c0, self.num_prototypes
        usage = torch.empty(n_cand, dtype=torch.float32, device=dev)
        nat.usage(usage, bank.use_cnt[c0:], bank.life_cnt[c0:], n_cand)
        _, top = torch.topk(usage, k=p, dim=-1, sorted=True)
        src = (top + c0).to(torch.int32)
        proto_key = torch.empty(p, self.CK, dtype=torch.float32, device=dev)
        proto_sel = torch.empty(p, self.CK, dtype=torch.float32, device=dev)
        nat.gather_rows(proto_key, bank.raw_key, src, p, self.CK * 4)
        nat.gather_rows(proto_sel, bank.raw_sel, src, p, self.CK * 4)
        q_hi, q_lo, bsq = self._pack_query(proto_key, proto_sel, 1, self.CK, p, 'co_')

        w0, lead, n_window = bank.window(c0, c1)
        ld = (n_window + 7) // 8 * 8
        sim_ws = self._buf('co_sim', (p, ld), torch.float32, dev)
        aff = self._buf('co_aff', (p, ld), torch.float16, dev)
        aff.zero_()
        proto_shr = torch.empty(p, dtype=torch.float32, device=dev)
        nat.sim_dense_softmax(bank.k_hi[w0:], bank.k_lo[w0:], bank.neg_s[w0:], bank.raw_shr[w0:], n_window, lead,
                              q_hi, q_lo, bsq, p, self.CK, sim_ws, ld, aff, ld, proto_shr)
        live = bank.objects
        proto_val = torch.empty(len(live) * self.CV, p, dtype=torch.float32, device=dev)
        for i in range(0, len(live), nat.MAX_GROUPS):
            part = live[i:i + nat.MAX_GROUPS]
            nat.readout(bank.values[:, :, w0:], bank.cap, bank.values.shape[0] * self.CV,
                        [bank.slot_of[o] * self.CV for o in part], [(i + j) * self.CV for j in range(len(part))],
                        self.CV, aff, ld, n_window, p, proto_val, p)
        return proto_key, proto_val, proto_shr

    def purge_except(self, obj_keep_idx: List[int]) -> None:
        """Forget every object not listed (memory_manager.py:220-229)."""
        keep = set(obj_keep_idx)
        for b in list(self._banks.keys()):
            self._banks[b].keep_objects(keep)
            if not self._banks[b].objects:
                del self._banks[b]
        if self._sensory_block is not None:
            rows = [i for i, o in enumerate(self._sensory_ids) if o in keep]
            self._sensory_block = self._sensory_block[rows].contiguous() if rows else None
            self._sensory_ids = [self._sensory_ids[i] for i in rows]
        if not self._banks:
            self.engaged = False

    def _long_term_mem_available(self) -> bool:
        return self.use_long_term and self.long_mem.engaged()

    # ------------------------------------------------------------------ sensory memory
    @property
    def sensory(self) -> Dict[int, torch.Tensor]:
        return {o: self._sensory_block[i] for i, o in enumerate(self._sensory_ids)}

    def initialize_sensory_if_needed(self, sample_key: torch.Tensor, ids: List[int]):
        new = [o for o in ids if o not in self._sensory_ids]
        if not new:
            return
        h, w = sample_key.shape[-2:]
        fresh = torch.zeros((len(new), self.sensory_dim, h, w), device=sample_key.device)
        self._sensory_block = fresh if self._sensory_block is None else torch.cat([self._sensory_block, fresh], 0)
        self._sensory_ids = self._sensory_ids + new

    def update_sensory(self, sensory: torch.Tensor, ids: List[int]):
        """sensory [1,K,C,h,w] in ``ids`` order; adopted without a copy when it covers every object."""
        if list(ids) == self._sensory_ids:
            self._sensory_block = sensory[0]
            return
        for j, o in enumerate(ids):
            self._sensory_block[self._sensory_ids.index(o)] = sensory[0, j]

    def get_sensory(self, ids: List[int]):
        """[1,K,C,h,w]; a view of the resident block when ``ids`` is the full object list."""
        if list(ids) == self._sensory_ids:
            return self._sensory_block.unsqueeze(0)
        rows = [self._sensory_ids.index(o) for o in ids]
        return self._sensory_block[rows].unsqueeze(0)
