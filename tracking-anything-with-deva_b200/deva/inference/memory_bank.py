"""Preallocated, token-major memory bank of one object bucket, resident in HBM.

Replaces the dict-of-growing-tensors of the reference (deva/inference/kv_memory_store.py:4-33,
one ``torch.cat`` of the whole bank per memory frame) with fixed buffers and O(new tokens) updates.

Physical layout of every per-token array (capacity ``cap`` tokens)::

        0 ........ lo ............... base ................. hi ........ cap
                    |<- long-term, ->|<--- working memory --->|
                    |  newest first  |      oldest first      |

The long-term region grows downwards from ``base`` and the working region upwards, so the valid
window ``[lo, hi)`` is always contiguous and a memory read is ONE similarity/top-k pass and ONE
readout GEMM over it - no concatenation of long-term and working tensors (memory_manager.py:107-113),
no stacking of per-object values (:83-89).  Slot order inside the long-term region is the reverse of
the reference's; top-k, softmax and readout are order independent, so only fp summation order
differs.

Per token: packed fp16 key rows (hi, lo) for the wgmma similarity GEMM, -shrinkage/sqrt(CK),
fp32 copies of key / selection / shrinkage (API views, consolidation), usage counters.
Per object: a [CV, cap] fp16 value matrix (memory-slot axis contiguous = K-major GEMM operand).
"""
from typing import Dict, List, Optional

import torch

from deva import _native as nat


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class BucketBank:
    def __init__(self, objects: List[int], ck: int, cv: int, long_cap: int, work_cap: int,
                 device: torch.device):
        self.objects: List[int] = list(objects)
        self.slot_of: Dict[int, int] = {o: i for i, o in enumerate(objects)}
        self.ck, self.cv = ck, cv
        self.device = device
        self.base = _round_up(long_cap, 8)
        self.cap = _round_up(self.base + work_cap, 8)
        self.lo = self.base
        self.hi = self.base
        # slot numbering epoch: bumped whenever existing tokens move (compaction, prepend, re-allocation).  The memory
        # read keeps each query's previous top-k slots per bank (temporal warm start of the streaming top-k) and may only
        # reuse them while the numbering is unchanged; appends keep it.
        self.numbering = 0
        self.read_idx = None   # int32 [q, 32]: slots the last read selected, relative to its window start
        self.read_key = None
        self._alloc(self.cap)

    # ------------------------------------------------------------------ storage
    def _alloc(self, cap: int) -> None:
        dev, ck = self.device, self.ck
        self.k_hi = torch.zeros(cap, 2 * ck, dtype=torch.float16, device=dev)
        self.k_lo = torch.zeros(cap, 2 * ck, dtype=torch.float16, device=dev)
        self.neg_s = torch.zeros(cap, dtype=torch.float32, device=dev)
        self.raw_key = torch.zeros(cap, ck, dtype=torch.float32, device=dev)
        self.raw_sel = torch.zeros(cap, ck, dtype=torch.float32, device=dev)
        self.raw_shr = torch.zeros(cap, dtype=torch.float32, device=dev)
        self.use_cnt = torch.zeros(cap, dtype=torch.float32, device=dev)
        self.life_cnt = torch.zeros(cap, dtype=torch.float32, device=dev)
        self.values = torch.zeros(len(self.slot_of), self.cv, cap, dtype=torch.float16, device=dev)

    _TOKEN_ARRAYS = ('k_hi', 'k_lo', 'neg_s', 'raw_key', 'raw_sel', 'raw_shr', 'use_cnt', 'life_cnt')

    def _grow(self, extra_long: int, extra_work: int) -> None:
        """Rare: capacity exceeded (long-term disabled, or config changed).  Re-centre into bigger buffers."""
        old = {n: getattr(self, n) for n in self._TOKEN_ARRAYS}
        old_values, old_base, old_lo, old_hi = self.values, self.base, self.lo, self.hi
        new_base = _round_up(old_base + extra_long, 8)
        new_cap = _round_up(new_base + (self.cap - old_base) + extra_work, 8)
        self.base, self.cap = new_base, new_cap
        self._alloc(new_cap)
        shift = new_base - old_base
        self.numbering += 1
        self.lo, self.hi = old_lo + shift, old_hi + shift
        for n, t in old.items():
            getattr(self, n)[self.lo:self.hi] = t[old_lo:old_hi]
        self.values[:, :, self.lo:self.hi] = old_values[:, :, old_lo:old_hi]

    # ------------------------------------------------------------------ sizes / window
    @property
    def long_size(self) -> int:
        return self.base - self.lo

    @property
    def work_size(self) -> int:
        return self.hi - self.base

    def window(self, start: Optional[int] = None, end: Optional[int] = None):
        """(w0, lead, n_window) of physical range [start, end) with w0 aligned down to 8 tokens."""
        start = self.lo if start is None else start
        end = self.hi if end is None else end
        w0 = start & ~7
        return w0, start - w0, end - w0

    # ------------------------------------------------------------------ append
    def _write_tokens(self, pos: int, key, selection, stride_c, stride_t, shrinkage, n: int) -> None:
        nat.pack_keys(key, selection, stride_c, stride_t, shrinkage, self.ck, n, self.k_hi[pos:], self.k_lo[pos:],
                      self.neg_s[pos:], self.raw_key[pos:], self.raw_sel[pos:] if selection is not None else None,
                      self.raw_shr[pos:])
        self.use_cnt[pos:pos + n] = 0
        self.life_cnt[pos:pos + n] = 1e-7  # kv_memory_store.py:94

    def append_work(self, key: torch.Tensor, shrinkage: torch.Tensor, selection: Optional[torch.Tensor],
                    values: Dict[int, torch.Tensor]) -> None:
        """key/selection: fp32 [CK, n] views (channel-major or token-major strides), shrinkage [n],
        values {obj: [CV, n]}: fp32 channel-major, or fp16 token-major views (NHWC encoder output)
        (kv_memory_store.py:97-116)."""
        n = key.shape[1]
        if self.hi + n > self.cap:
            self._grow(0, max(n, self.cap - self.base))
        assert selection is None or selection.stride() == key.stride()
        self._write_tokens(self.hi, key, selection, key.stride(0), key.stride(1), shrinkage, n)
        for obj, v in values.items():
            dst = self.values[self.slot_of[obj], :, self.hi:]
            if v.dtype == torch.float16 and v.stride(0) == 1 and v.stride(1) == self.cv:
                nat.transpose_append(v, dst, self.cap, n, self.cv)
            else:
                if v.dtype != torch.float32 or v.stride(1) != 1:
                    v = v.float().contiguous()
                nat.append_values(v, v.stride(0), dst, self.cap, self.cv, n)
        self.hi += n

    def prepend_long(self, key_rows: torch.Tensor, shrinkage: torch.Tensor, values: torch.Tensor) -> None:
        """key_rows [n, CK] token-major, shrinkage [n], values [len(objects)*CV, n] in slot order."""
        n = key_rows.shape[0]
        if self.lo - n < 0:
            self._grow(max(n, self.base), 0)
        pos = self.lo - n
        self.numbering += 1
        self._write_tokens(pos, key_rows, None, 1, self.ck, shrinkage, n)
        live = [self.slot_of[o] for o in self.objects]
        for i, slot in enumerate(live):
            nat.append_values(values[i * self.cv:], values.stride(0), self.values[slot, :, pos:], self.cap, self.cv, n)
        self.lo = pos

    # ------------------------------------------------------------------ compaction
    def _compact(self, src_idx: torch.Tensor, dst_start: int) -> None:
        """Move tokens src_idx (physical, int32, ascending) to [dst_start, dst_start+len) via scratch copies."""
        n = int(src_idx.numel())
        self.numbering += 1
        if n == 0:
            return
        for name in ('k_hi', 'k_lo', 'raw_key', 'raw_sel'):
            arr = getattr(self, name)
            tmp = torch.empty(n, arr.shape[1], dtype=arr.dtype, device=self.device)
            nat.gather_rows(tmp, arr, src_idx, n, arr.shape[1] * arr.element_size())
            arr[dst_start:dst_start + n] = tmp
        for name in ('neg_s', 'raw_shr', 'use_cnt', 'life_cnt'):
            arr = getattr(self, name)
            tmp = torch.empty(n, dtype=torch.float32, device=self.device)
            nat.gather_f32(tmp, arr, src_idx, n)
            arr[dst_start:dst_start + n] = tmp
        rows = self.values.shape[0] * self.cv
        tmp = torch.empty(rows, n, dtype=torch.float16, device=self.device)
        nat.gather_cols_f16(tmp, n, self.values, self.cap, src_idx, rows, n)
        self.values.view(rows, self.cap)[:, dst_start:dst_start + n] = tmp

    def drop_work_range(self, start: int, end: int) -> None:
        """Keep working tokens [0, start) and [W+end, W) (end < 0): KeyValueMemoryStore.sieve_by_range."""
        w = self.work_size
        tail = -end
        src = torch.arange(self.base + w - tail, self.base + w, dtype=torch.int32, device=self.device)
        self._compact(src, self.base + start)
        self.hi = self.base + start + tail

    def evict_long(self, max_size: int) -> None:
        """remove_obsolete_features (kv_memory_store.py:164-185) on the long-term region."""
        n = self.long_size
        usage = torch.empty(n, dtype=torch.float32, device=self.device)
        nat.usage(usage, self.use_cnt[self.lo:], self.life_cnt[self.lo:], n)
        smallest, _ = torch.topk(usage, k=n - max_size, largest=False, sorted=True)
        keep = torch.nonzero(usage > smallest[-1]).reshape(-1).to(torch.int32) + self.lo  # strict '>' (quirk Q5)
        kept = int(keep.numel())
        self._compact(keep, self.base - kept)
        self.lo = self.base - kept

    # ------------------------------------------------------------------ objects
    def keep_objects(self, keep_ids) -> None:
        self.objects = [o for o in self.objects if o in keep_ids]

    # ------------------------------------------------------------------ reference-shaped views
    def key_view(self, kind: str) -> torch.Tensor:
        a, b = (self.lo, self.base) if kind == 'long' else (self.base, self.hi)
        return self.raw_key[a:b].t()

    def shrinkage_view(self, kind: str) -> torch.Tensor:
        a, b = (self.lo, self.base) if kind == 'long' else (self.base, self.hi)
        return self.raw_shr[a:b].unsqueeze(0)

    def selection_view(self, kind: str) -> torch.Tensor:
        a, b = (self.lo, self.base) if kind == 'long' else (self.base, self.hi)
        return self.raw_sel[a:b].t()

    def value_view(self, obj: int, kind: str) -> torch.Tensor:
        a, b = (self.lo, self.base) if kind == 'long' else (self.base, self.hi)
        return self.values[self.slot_of[obj], :, a:b]
