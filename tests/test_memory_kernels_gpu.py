"""The memory read, consolidation and bank-compaction kernels (csrc/simtopk.cu, readout.cu, bank_ops.cu) against float64
references, in the states the memory manager puts a bank in.

A read runs on a window of the bank (``BucketBank.window()``): an 8-aligned start w0 inside larger buffers, 1..7 lead
slots that belong to no memory, a long-term region and the working region.  The read counts usage and life in one or
both regions, reads values through object row maps with gaps (``slot_of[o] * CV`` against ``order[o] * CV``), and may
be warm-started from the previous frame's selection.  Consolidation reads 128 prototypes, gathered from the bank's own
slots, against a whole window of candidates.

Every output is a view of a NaN-filled buffer followed by a guard region, and every window-sliced operand has NaN key
rows in its lead slots and NaN everywhere past the window (lead value columns stay finite: the read-out multiplies them
by zero weights).  References are float64 on the device and reuse oracle/memory_math.py; kernels whose result is fixed
by their operands (copies, fp16 conversion, one add into zero, the same fp16 tile fed to the same GEMM) are compared bit
for bit.  Each check prints its measured error beside its bound.
"""
import math

import numpy as np
import pytest
import torch

from oracle import memory_math as mm

gpu = pytest.mark.gpu
CK = 64
LP = 32            # row pitch of the top-k lists (deva._native.LIST_PITCH)
GUARD = 64
I32_FILL = -0x5A5A5A5A
READ_REL = 2.0 ** -16   # read-out bound, relative to sum_j |w_j v_j| (derivation in _check_readout)
SIM_ABS = 1e-4          # similarity bound (chosen: the existing memory-read tests' value)
W_ABS = 2e-5            # softmax weight bound over the selected slots (chosen: the existing memory-read tests' value)


def _nat():
    from deva import _native
    _native.require_device()
    return _native


def _report(name, err, bound):
    print(f'[memory-kernels] {name}: max err {err:.3e}, bound {bound:.3e}')


class Outputs:
    """Tensors as views of larger buffers filled with NaN (int32: I32_FILL), each followed by a guard region."""

    def __init__(self):
        self.bufs = []

    def new(self, shape, dtype, data=None):
        n = math.prod(shape)
        buf = torch.empty(n + GUARD, dtype=dtype, device='cuda')
        buf.fill_(I32_FILL if dtype == torch.int32 else float('nan'))
        if data is not None:
            buf[:n] = data.reshape(-1)
        self.bufs.append((buf, n))
        return buf[:n].view(shape)

    def check_guards(self):
        for buf, n in self.bufs:
            g = buf[n:]
            ok = (g == I32_FILL).all() if buf.dtype == torch.int32 else torch.isnan(g).all()
            assert bool(ok), 'a kernel wrote past its output'


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _keys(g, n, q, rows):
    mk = torch.randn(CK, n, generator=g, device='cuda')
    ms = 1 + torch.rand(n, generator=g, device='cuda')
    qk = torch.randn(CK, q, generator=g, device='cuda')
    qe = torch.sigmoid(torch.randn(CK, q, generator=g, device='cuda'))
    mv = torch.randn(rows, n, generator=g, device='cuda')
    return mk, ms, qk, qe, mv


class Window:
    """A bank window as BucketBank.window() hands it to the kernels.  Buffers hold `cap` slots; window slot i is buffer
    slot w0 + i (w0 8-aligned); slots [0, lead) of the window are alignment lead, [lead, lead + n_long) long-term and
    the rest working memory.  Lead key rows and everything past the window are NaN; lead value columns are finite."""

    def __init__(self, nat, mk, ms, mv, lead, n_long=0, w0=40, tail=88):
        n = mk.shape[1]
        self.n, self.lead, self.w0 = n, lead, w0
        self.nw = lead + n
        self.n_long = lead + n_long  # the kernels' n_long: window slots below it are long-term memory
        self.cap = cap = (w0 + self.nw + tail + 7) // 8 * 8
        nan, dev = float('nan'), 'cuda'
        self.k_hi = torch.full((cap, 2 * CK), nan, dtype=torch.float16, device=dev)
        self.k_lo = torch.full_like(self.k_hi, nan)
        self.neg_s = torch.full((cap, ), nan, device=dev)
        self.raw_key = torch.full((cap, CK), nan, device=dev)
        self.raw_shr = torch.full((cap, ), nan, device=dev)
        s = w0 + lead
        self.raw_shr[w0:s] = 1.0  # multiplied by zero probabilities, like the lead value columns
        nat.pack_keys(mk.contiguous(), None, n, 1, ms.contiguous(), CK, n, self.k_hi[s:], self.k_lo[s:], self.neg_s[s:],
                      self.raw_key[s:], None, self.raw_shr[s:])
        self.rows = mv.shape[0]
        self.values = torch.full((self.rows, cap), nan, dtype=torch.float16, device=dev)
        self.values[:, w0:s] = 1.0
        nat.append_values(mv.contiguous(), n, self.values[:, s:], cap, self.rows, n)
        self.mk, self.ms = mk, ms

    def keys(self):
        return self.k_hi[self.w0:], self.k_lo[self.w0:], self.neg_s[self.w0:]

    def vals(self):
        return self.values[:, self.w0:]

    def sim64(self, qk, qe):
        """fp64 similarity [n_window - lead, q] of the window's memory slots."""
        return mm.similarity(self.mk.double(), self.ms.double(), qk.double(), qe.double())


def _pack_q(nat, qk, qe, token_major=False):
    """qk/qe: [CK, q] (channel-major) or, token_major, [q, CK] rows."""
    q = qk.shape[0] if token_major else qk.shape[1]
    q_hi = torch.empty(q, 2 * CK, dtype=torch.float16, device='cuda')
    q_lo = torch.empty_like(q_hi)
    bsq = torch.empty(q, device='cuda')
    sc, sq = (1, CK) if token_major else (q, 1)
    nat.pack_query(qk.contiguous(), qe.contiguous(), sc, sq, CK, q, q_hi, q_lo, bsq)
    return q_hi, q_lo, bsq


def _topk(nat, win, packed, q, top_k, outs, aff=None, ldp=0, use=None, life=None, count_long=False, count_work=False,
          prev=None):
    kh, kl, ns = win.keys()
    ws = torch.empty(nat.simtopk_workspace_bytes(q), dtype=torch.uint8, device='cuda')
    idx = outs.new((q, LP), torch.int32)
    w = outs.new((q, LP), torch.float32)
    thr = outs.new((q, ), torch.float32) if prev is not None else None
    nat.sim_topk(kh, kl, ns, win.nw, win.lead, *packed, q, CK, top_k, ws, idx, w, aff, ldp, use, life, win.n_long,
                 count_long, count_work, prev_idx=prev, thr_ws=thr)
    return idx, w, thr


# ------------------------------------------------------------------------------------------------- references
def ranked(sim, k):
    """The tie rule: the first k slots under (similarity descending, slot ascending); sim [n, q] -> [q, k] slots."""
    return torch.sort(sim, dim=0, descending=True, stable=True)[1][:k].t()


def dense_affinity(idx, w, top_k, n):
    """fp64 [q, n] affinity of (idx, w) lists with the weights rounded to fp16, as both read-out kernels consume them."""
    a = torch.zeros(idx.shape[0], n, dtype=torch.float64, device=idx.device)
    return a.scatter_add_(1, idx[:, :top_k].long(), w[:, :top_k].half().double())


def readout_ref(values, val_row, rows_per_group, aff):
    """Row-mapped read-out in fp64: group g's rows values[val_row[g] + r] times aff^T, stacked in call order, and the
    magnitude sum_n |v w| that bounds the fp32 accumulation error."""
    v = torch.cat([values[r:r + rows_per_group] for r in val_row]).double()
    return v @ aff.t(), v.abs() @ aff.abs().t()


def clustered_lists(q, top_k, n_window, lead, plans, seed):
    """(idx, w) int32 / fp32 [q, 32] whose 256-query tiles each put all their entries into one or two 64-slot k-blocks.
    plans[t % len(plans)] = (block a, entries in a, block b): the tile's other entries go to block b.  Returns the
    lists and {(tile, block): entries}."""
    rng = np.random.default_rng(seed)
    idx = np.zeros((q, LP), np.int32)
    w = np.zeros((q, LP), np.float32)
    counts = {}
    for t in range(-(-q // 256)):
        q0, nq = t * 256, min(256, q - t * 256)
        a, ca, b = plans[t % len(plans)]
        total = nq * top_k
        ca = min(ca, total)
        labels = np.array([a] * ca + [b] * (total - ca))
        for blk in (a, b):
            if (labels == blk).any():
                counts[(t, blk)] = int((labels == blk).sum())
        for ql in range(nq):
            mine = labels[ql::nq][:top_k]  # entry e of the tile goes to query e % nq
            row = []
            for blk in np.unique(mine):
                lo, hi = max(blk * 64, lead), min(blk * 64 + 64, n_window)
                row += list(rng.choice(np.arange(lo, hi), size=int((mine == blk).sum()), replace=False))
            idx[q0 + ql, :top_k] = row
            x = rng.random(top_k) + 0.1
            w[q0 + ql, :top_k] = x / x.sum()
    return torch.from_numpy(idx), torch.from_numpy(w), counts


def merge_ref(vals, ids, top_k, q):
    """The documented merge rule: per query the top_k valid (idx >= 0) candidates under (value descending, slot
    ascending), then a softmax over them; vals/ids [n_lists][32][q_pitch].  -> idx int64, w fp64, sim fp32 [q, 32]."""
    out_i = np.zeros((q, LP), np.int64)
    out_w = np.zeros((q, LP), np.float64)
    out_s = np.full((q, LP), -np.inf, np.float32)
    for i in range(q):
        v = vals[:, :top_k, i].reshape(-1)
        s = ids[:, :top_k, i].reshape(-1)
        ok = s >= 0
        v, s = v[ok], s[ok]
        order = np.lexsort((s, -v.astype(np.float64)))[:top_k]
        m = len(order)
        out_i[i, :m], out_s[i, :m] = s[order], v[order]
        e = np.exp(v[order].astype(np.float64) - float(v[order][0]))
        out_w[i, :m] = e / e.sum()
    return out_i, out_w, out_s


# ------------------------------------------------------------------------------------------------- shared checks
def _check_selection(idx, w, sim, top_k, lead, name):
    """The selection is valid and distinct, it is the fp64 top-k except where the k-th / (k+1)-th gap is under 2e-4,
    and its weights are the fp64 softmax of the selected slots."""
    q, n = idx.shape[0], sim.shape[0]
    assert bool((idx[:, top_k:] == 0).all()) and bool((w[:, top_k:] == 0).all())
    sel = idx[:, :top_k].long() - lead
    assert int(sel.min()) >= 0 and int(sel.max()) < n
    srt = torch.sort(sel, 1)[0]
    assert bool((srt[:, 1:] != srt[:, :-1]).all()), 'a slot was selected twice'
    vals = torch.sort(sim, 0, descending=True)[0]
    gap = (vals[top_k - 1] - vals[top_k]) if n > top_k else torch.full((q, ), 1.0, dtype=sim.dtype, device=sim.device)
    same = (torch.sort(ranked(sim, top_k), 1)[0] == srt).all(1)
    assert bool((same | (gap < 2e-4)).all()), f'{name}: top-k sets differ on {int((~same).sum())} queries'
    sel_sim = sim.t().gather(1, sel)
    assert bool((sel_sim[:, :-1] - sel_sim[:, 1:] > -2e-4).all()), 'not sorted by descending similarity'
    err = float((w[:, :top_k].double() - torch.softmax(sel_sim, 1)).abs().max())
    _report(f'{name} weights', err, W_ABS)
    assert err < W_ABS


def _check_readout(got, ref, mag, name):
    """fp16 operands are exact in fp32 products; the fp32 accumulation rounds once per 16-deep k-step that has a
    non-zero term (at most top_k <= 32 of them), each within one ulp of the running sum <= sum |w v|: 32 * 2^-23 =
    2^-18 of the magnitude.  READ_REL = 2^-16 leaves a factor 4 for the tensor core's internal alignment."""
    err = (got.double() - ref).abs()
    bound = READ_REL * mag + 1e-30
    worst = float((err / bound).max())
    _report(f'{name} read-out (err / bound)', worst, 1.0)
    assert worst <= 1.0, name


def _run_readouts(nat, win, idx, w, top_k, q, aff16, ldp, val_row, out_row, cv, n_out, ldo, name):
    """Dense and sparse read-out, fp32 and fp16 token-major, into NaN buffers: every called group's rows equal fp64,
    the two kernels agree bit for bit, fp16 is the fp32 result rounded, and rows of uncalled groups stay NaN."""
    outs = Outputs()
    rows = n_out * cv
    vals = win.vals()
    res = {}
    for kind in ('dense', 'sparse'):
        out = outs.new((rows, ldo), torch.float32)
        tok = outs.new((n_out, q, cv), torch.float16)
        for o, t in ((out, None), (None, tok)):
            if kind == 'dense':
                nat.readout(vals, win.cap, win.rows, val_row, out_row, cv, aff16, ldp, win.nw, q, o, ldo, t)
            else:
                rws = torch.empty(nat.readout_sparse_workspace_bytes(q, win.nw), dtype=torch.uint8, device='cuda')
                nat.readout_sparse(vals, win.cap, win.rows, val_row, out_row, cv, idx, w, top_k, win.nw, q, rws, o, ldo, t)
        res[kind] = (out, tok)
    torch.cuda.synchronize()
    outs.check_guards()
    ref, mag = readout_ref(vals[:, :win.nw], val_row, cv, dense_affinity(idx, w, top_k, win.nw))
    called = torch.zeros(n_out, dtype=torch.bool)
    for r in out_row:
        called[r // cv] = True
    dense, sparse = res['dense'], res['sparse']
    got_d = torch.cat([dense[0][r:r + cv, :q] for r in out_row])
    got_s = torch.cat([sparse[0][r:r + cv, :q] for r in out_row])
    _check_readout(got_d, ref, mag, name)
    # both kernels feed the same fp16 affinity tiles to the same wgmma sequence in the same k order
    assert torch.equal(got_d, got_s), f'{name}: sparse read-out differs from the dense one'
    for out, tok in (dense, sparse):
        o3 = out.view(n_out, cv, ldo)
        assert bool(torch.isnan(o3[~called]).all()), 'rows of a group outside the call were written'
        assert bool(torch.isnan(o3[:, :, q:]).all()), 'columns past q were written'
        assert bool(torch.isnan(tok[~called].float()).all()), 'token-major rows of a group outside the call were written'
        want = o3[called, :, :q].half().permute(0, 2, 1)
        assert torch.equal(tok[called], want), f'{name}: fp16 token-major output is not the rounded fp32 result'
    return dense[0]


# ------------------------------------------------------------------------------------------------- CPU: the references
def test_references_on_cpu():
    # tie rule: equal similarities are ranked by ascending slot
    sim = torch.tensor([[0.5, 1.0], [0.9, 1.0], [0.9, 0.2], [0.1, 1.0], [0.9, 0.3]], dtype=torch.float64)
    assert ranked(sim, 3).tolist() == [[1, 2, 4], [0, 1, 3]]
    assert ranked(sim, 2).tolist() == [[1, 2], [0, 1]]
    # clustered lists: the requested entry counts per (tile, block), more than 1024 in one block, distinct slots
    q, top_k, nw, lead = 256 * 11 + 77, 30, 64 * 20, 3
    idx, w, counts = clustered_lists(q, top_k, nw, lead, CLUSTER_PLANS, 1)
    for t in range(12):
        nq = min(256, q - 256 * t)
        a, ca, b = CLUSTER_PLANS[t % len(CLUSTER_PLANS)]
        ca = min(ca, nq * top_k)
        blocks = (idx[256 * t:256 * t + nq, :top_k].long() // 64).reshape(-1)
        assert int((blocks == a).sum()) == ca == counts[(t, a)]
        assert int((blocks == b).sum()) == nq * top_k - ca
    assert max(counts.values()) > 1024 and {64, 65, 1023, 1024, 1025} <= set(counts.values())
    s = torch.sort(idx[:, :top_k].long(), 1)[0]
    assert bool((s[:, 1:] != s[:, :-1]).all()) and int(idx[:, :top_k].min()) >= lead and int(idx.max()) < nw
    assert bool((w[:, :top_k] > 0).all()) and bool((w[:, top_k:] == 0).all())
    assert float((w.sum(1) - 1).abs().max()) < 1e-6
    # row-map reference against a per-query loop
    g = torch.Generator().manual_seed(2)
    values = torch.randn(5 * 128, 300, generator=g).half()
    il = torch.stack([torch.randperm(300, generator=g)[:7] for _ in range(20)]).int()
    wl = torch.rand(20, 7, generator=g)
    ref, mag = readout_ref(values, [384, 0], 128, dense_affinity(il, wl, 7, 300))
    for r, vr in enumerate([384, 0]):
        for j in range(20):
            want = sum(values[vr:vr + 128, int(il[j, e])].double() * float(wl[j, e].half()) for e in range(7))
            assert torch.allclose(ref[r * 128:(r + 1) * 128, j], want, rtol=1e-12, atol=1e-12)
    assert bool((mag >= ref.abs()).all())
    # merge rule: ties across lists go to the lower slot, empty entries are skipped, short rows are padded
    vals = np.full((2, LP, 1), np.nan, np.float32)
    ids = np.full((2, LP, 1), -1, np.int32)
    vals[0, :2, 0], ids[0, :2, 0] = [3.0, 1.0], [9, 4]
    vals[1, :2, 0], ids[1, :2, 0] = [3.0, 2.0], [5, 7]
    oi, ow, osim = merge_ref(vals, ids, 3, 1)
    assert oi[0, :4].tolist() == [5, 9, 7, 0] and osim[0, :3].tolist() == [3.0, 3.0, 2.0] and osim[0, 3] == -np.inf
    assert abs(ow[0, 0] - 1 / (2 + math.exp(-1))) < 1e-12 and ow[0, 3] == 0


# ------------------------------------------------------------------------------------------------- bank window
@gpu
@pytest.mark.parametrize('top_k,n,n_long,lead,q', [
    (1, 1500, 333, 5, 600),
    (7, 2600, 777, 1, 900),
    (30, 5000, 1013, 7, 1100),
    (32, 3000, 100, 4, 700),
    (30, 30, 11, 2, 300),     # n_window - n_lead == top_k: every slot is selected
    (32, 32, 13, 6, 257),
])
def test_window_with_long_term_region_counts_usage_per_region(top_k, n, n_long, lead, q):
    nat = _nat()
    g = _gen(top_k * 1000 + n)
    mk, ms, qk, qe, mv = _keys(g, n, q, 128)
    win = Window(nat, mk, ms, mv, lead, n_long)
    packed = _pack_q(nat, qk, qe)
    sim = win.sim64(qk, qe)
    use0 = (0.5 + 3 * torch.rand(win.cap, generator=g, device='cuda'))
    life0 = torch.randint(0, 40, (win.cap, ), generator=g, device='cuda').float() + 1e-7
    ldp = (win.nw + 7) // 8 * 8 + 16
    first = None
    for count_long in (False, True):
        for count_work in (False, True):
            outs = Outputs()
            use, life = outs.new((win.cap, ), torch.float32, use0), outs.new((win.cap, ), torch.float32, life0)
            aff = outs.new((q, ldp), torch.float16)
            idx, w, _ = _topk(nat, win, packed, q, top_k, outs, aff, ldp, use[win.w0:], life[win.w0:], count_long,
                              count_work)
            torch.cuda.synchronize()
            outs.check_guards()
            name = f'window k={top_k} n={n} long={count_long} work={count_work}'
            if first is None:
                first = (idx.clone(), w.clone())
                _check_selection(idx, w, sim, top_k, lead, name)
            else:  # the counters do not change the selection
                assert torch.equal(idx, first[0]) and torch.equal(w, first[1])
            # dense affinity rows: exactly the fp16 weights at the selected slots
            want = torch.zeros(q, ldp, dtype=torch.float16, device='cuda')
            want.scatter_(1, idx[:, :top_k].long(), w[:, :top_k].half())
            assert torch.equal(aff, want)
            # counted region [lo, hi) of the window: usage += fp64 affinity column sums, life += 1; all else untouched
            lo = lead if count_long else win.n_long
            hi = win.nw if count_work else win.n_long
            s = slice(win.w0 + lo, win.w0 + max(lo, hi))
            add = torch.zeros(win.cap, dtype=torch.float64, device='cuda')
            add.index_add_(0, idx[:, :top_k].reshape(-1).long() + win.w0, w[:, :top_k].reshape(-1).double())
            cnt = torch.zeros(win.cap, dtype=torch.float64, device='cuda')
            cnt.index_add_(0, idx[:, :top_k].reshape(-1).long() + win.w0,
                           torch.ones(q * top_k, dtype=torch.float64, device='cuda'))
            want_use = use0.double() + add
            # fp32 accumulation of cnt terms onto the start value: each add rounds by <= 2^-24 of the running sum
            bound = (cnt + 1) * 2.0 ** -24 * want_use
            err = (use.double() - want_use).abs()
            _report(f'{name} usage', float(err[s].max()) if hi > lo else 0.0, float(bound[s].max()) if hi > lo else 0.0)
            assert bool((err[s] <= bound[s]).all()) and float(err[s].max() if hi > lo else 0) < 1e-4
            assert torch.equal(life[s], life0[s] + 1), 'life must be start + 1 in the counted region'
            keep = torch.ones(win.cap, dtype=torch.bool, device='cuda')
            keep[s] = False
            assert torch.equal(use[keep], use0[keep]) and torch.equal(life[keep], life0[keep]), \
                'a counter outside the counted region changed'
    idx, w = first
    aff16 = torch.zeros(q, ldp, dtype=torch.float16, device='cuda').scatter_(1, idx[:, :top_k].long(),
                                                                              w[:, :top_k].half())
    aff16[:, win.nw:] = float('nan')
    _run_readouts(nat, win, idx, w, top_k, q, aff16, ldp, [0], [0], 128, 1, q, f'window k={top_k} n={n}')


# ------------------------------------------------------------------------------------------------- object row maps
@gpu
@pytest.mark.parametrize('groups,cv,q,ld_pad', [
    (1, 128, 1000, 0),
    (5, 256, 700, 1),      # odd ld_out: the scalar store path
    (16, 512, 513, 0),
    (5, 512, 128, 0),      # consolidation: 128 prototypes (under one 256-query tile), compact output rows
])
def test_object_row_maps(groups, cv, q, ld_pad):
    nat = _nat()
    g = _gen(groups * 7 + cv)
    slots, n, lead, top_k = 20, 2037, 3, 30
    mk, ms, qk, qe, mv = _keys(g, n, q, slots * cv)
    win = Window(nat, mk, ms, mv, lead, n_long=300)
    packed = _pack_q(nat, qk, qe)
    ldp = (win.nw + 7) // 8 * 8 + 16
    outs = Outputs()
    aff = outs.new((q, ldp), torch.float16)
    idx, w, _ = _topk(nat, win, packed, q, top_k, outs, aff, ldp)
    torch.cuda.synchronize()
    aff[:, win.nw:] = float('nan')
    compact = q == 128
    n_out = groups if compact else groups + 3
    val_row = [int(s) * cv for s in torch.randperm(slots, generator=g, device='cuda')[:groups]]
    out_row = [j * cv for j in range(groups)] if compact else \
        [int(s) * cv for s in torch.randperm(n_out, generator=g, device='cuda')[:groups]]
    _run_readouts(nat, win, idx, w, top_k, q, aff, ldp, val_row, out_row, cv, n_out, q + ld_pad,
                  f'row maps G={groups} cv={cv} q={q}')


# ------------------------------------------------------------------------------------------------- clustered selections
# (block a, entries in block a, block b) per 256-query tile: the heavy and light blocks of a tile are 4 k-blocks apart,
# so in a CTA's k-loop the same pipeline stage serves both; the counts straddle the 64-entry prefetch and the
# 1024-entry record of scattered offsets (above it the next use of the stage clears the whole tile)
CLUSTER_PLANS = [(2, 1025, 6), (6, 64, 10), (10, 7680, 14), (3, 1024, 7), (7, 65, 11), (11, 1023, 15),
                 (15, 7615, 19), (0, 4000, 4), (12, 7680, 16), (1, 2000, 5), (9, 6656, 13)]


@gpu
def test_clustered_selections_sparse_equals_dense():
    nat = _nat()
    g = _gen(31)
    top_k, lead, cv, groups = 30, 3, 512, 5
    nw = 64 * 20
    q = 256 * 11 + 77  # 12 query tiles x 20 row tiles: more tiles than SMs, so CTAs reuse stages across tiles
    idx, w, counts = clustered_lists(q, top_k, nw, lead, CLUSTER_PLANS, 5)
    assert max(counts.values()) > 1024
    mk, ms, _, _, mv = _keys(g, nw - lead, 1, groups * cv)
    win = Window(nat, mk, ms, mv, lead)
    idx, w = idx.cuda(), w.cuda()
    ldp = nw + 16
    aff = torch.zeros(q, ldp, dtype=torch.float16, device='cuda').scatter_(1, idx[:, :top_k].long(), w[:, :top_k].half())
    aff[:, nw:] = float('nan')
    _run_readouts(nat, win, idx, w, top_k, q, aff, ldp, [int(i) * cv for i in (3, 0, 4, 1, 2)],
                  [int(i) * cv for i in (1, 4, 0, 2, 3)], cv, groups, q, 'clustered')


# ------------------------------------------------------------------------------------------------- consolidation
@gpu
@pytest.mark.parametrize('n,lead', [(8100, 3), (40800, 5)])
def test_consolidation_dense_softmax(n, lead):
    nat = _nat()
    g = _gen(n)
    p = 128
    mk, ms, _, _, _ = _keys(g, n, 1, 1)
    sel = torch.sigmoid(torch.randn(CK, n, generator=g, device='cuda'))
    win = Window(nat, mk, ms, torch.zeros(1, n, device='cuda'), lead)
    raw_sel = torch.full((win.cap, CK), float('nan'), device='cuda')
    raw_sel[win.w0 + lead:win.w0 + win.nw] = sel.t()
    # prototypes: memory slots themselves, gathered from the bank's token-major rows and packed token-major
    src = (torch.randperm(n, generator=g, device='cuda')[:p] + win.w0 + lead).int()
    outs = Outputs()
    pk, ps = outs.new((p, CK), torch.float32), outs.new((p, CK), torch.float32)
    nat.gather_rows(pk, win.raw_key, src, p, CK * 4)
    nat.gather_rows(ps, raw_sel, src, p, CK * 4)
    packed = _pack_q(nat, pk, ps, token_major=True)
    ld = (win.nw + 7) // 8 * 8 + 8
    sim_ws = outs.new((p, ld), torch.float32)
    aff = outs.new((p, ld), torch.float16)
    shr_out = outs.new((p, ), torch.float32)
    kh, kl, ns = win.keys()
    nat.sim_dense_softmax(kh, kl, ns, win.raw_shr[win.w0:], win.nw, lead, *packed, p, CK, sim_ws, ld, aff, ld, shr_out)
    torch.cuda.synchronize()
    outs.check_guards()
    slot = src.long() - win.w0 - lead
    assert torch.equal(pk, mk.t()[slot]) and torch.equal(ps, sel.t()[slot])
    sim = mm.similarity(mk.double(), ms.double(), pk.t().double(), ps.t().double()).t()  # [p, n]
    assert float(sim.max(1)[0].abs().max()) < 1e-3, 'each prototype row peaks at its own slot (similarity ~0)'
    err = float((sim_ws[:, lead:win.nw].double() - sim).abs().max())
    _report(f'consolidation n={n} similarity', err, SIM_ABS)
    assert err < SIM_ABS
    assert bool((sim_ws[:, :lead] == float('-inf')).all()) and bool((aff[:, :lead] == 0).all())
    assert bool(torch.isnan(sim_ws[:, win.nw:]).all()) and bool(torch.isnan(aff[:, win.nw:].float()).all())
    # softmax: a similarity error <= SIM_ABS moves each probability by a factor within exp(+-2 SIM_ABS); fp32 sums of
    # <= 40800 terms add ~2e-5 relative; the fp16 store rounds by 2^-11 relative (2^-25 absolute below 2^-14)
    p64 = torch.softmax(sim, 1)
    rel = 2 * SIM_ABS + 2e-5
    perr = (aff[:, lead:win.nw].double() - p64).abs()
    pbound = p64 * (2.0 ** -11 + rel) + 2.0 ** -25
    _report(f'consolidation n={n} softmax (err / bound)', float((perr / pbound).max()), 1.0)
    assert bool((perr <= pbound).all())
    shr64 = p64 @ ms.double()
    serr = float(((shr_out.double() - shr64).abs() / shr64).max())
    _report(f'consolidation n={n} shrinkage read-out (relative)', serr, rel)
    assert serr < rel


# ------------------------------------------------------------------------------------------------- exact ties
@gpu
@pytest.mark.parametrize('frame,q', [
    (1000, 2000),   # 4 splits of the memory axis: the copies of a token land in different candidate lists
    (1024, 8448),   # one split, frame a multiple of 128 slots: all copies of a token land in the same list
])
def test_exact_ties_follow_the_tie_rule(frame, q):
    """A bank holding one frame 4 times (duplicated video frames): bit-identical keys and values.  top_k = 30 is not a
    multiple of 4, so every query has a boundary token of which only 2 copies are selected: the lower slots."""
    nat = _nat()
    g = _gen(frame + q)
    top_k, lead, copies = 30, 5, 4
    mkf, msf, qk, qe, mvf = _keys(g, frame, q, 128)
    win = Window(nat, mkf.repeat(1, copies), msf.repeat(copies), mvf.repeat(1, copies), lead)
    packed = _pack_q(nat, qk, qe)
    outs = Outputs()
    idx, w, _ = _topk(nat, win, packed, q, top_k, outs)
    idx2, w2, _ = _topk(nat, win, packed, q, top_k, outs)
    warm, warm_w, thr = _topk(nat, win, packed, q, top_k, outs, prev=idx.clone())
    torch.cuda.synchronize()
    outs.check_guards()
    assert torch.equal(idx, idx2) and torch.equal(w, w2), 'the same read gave two results'
    assert torch.equal(warm, idx) and torch.equal(warm_w, w), 'cold and warm-started reads differ'
    assert bool(torch.isfinite(thr).all())
    sel = idx[:, :top_k].long() - lead
    srt = torch.sort(sel, 1)[0]
    assert int(sel.min()) >= 0 and int(sel.max()) < copies * frame
    assert bool((srt[:, 1:] != srt[:, :-1]).all()), 'a slot was selected twice'
    # every query: of each token, the selected copies are the lowest ones, and exactly one token is cut at the boundary
    tok, cop = sel % frame, sel // frame
    per = torch.zeros(q, frame, dtype=torch.long, device='cuda').scatter_add_(1, tok, torch.ones_like(tok))
    cmax = torch.zeros(q, frame, dtype=torch.long, device='cuda').scatter_reduce_(1, tok, cop, 'amax')
    chosen = per > 0
    assert bool((cmax[chosen] == per[chosen] - 1).all()), 'a tie was resolved to a higher slot'
    assert bool(((per == 2).sum(1) == 1).all()) and bool(((per == 4).sum(1) == 7).all())
    # queries whose top 9 distinct similarities are 2e-4 apart: the exact sequence under (sim desc, slot asc)
    simf = mm.similarity(mkf.double(), msf.double(), qk.double(), qe.double())
    top9 = torch.sort(simf, 0, descending=True)[0][:9]
    clean = ((top9[:-1] - top9[1:]) > 2e-4).all(0)
    assert int(clean.sum()) > q // 2
    want = ranked(simf.repeat(copies, 1), top_k)
    assert torch.equal(sel[clean], want[clean])
    sel_sim = simf.repeat(copies, 1).t().gather(1, sel)
    err = float((w[:, :top_k].double() - torch.softmax(sel_sim, 1)).abs().max())
    _report(f'ties frame={frame} weights', err, W_ABS)
    assert err < W_ABS


# ------------------------------------------------------------------------------------------------- warm start
@gpu
def test_warm_start_with_repeated_slots_is_exact():
    """prev_idx rows that repeat a slot are not top_k distinct slots: their minimum similarity is no lower bound of
    the k-th best, and they must not gate anything out.  Each query has 29 near slots and a 30th far below them."""
    nat = _nat()
    g = _gen(77)
    q, near, far, top_k, lead = 300, 29, 2000, 30, 3
    qk = torch.randn(CK, q, generator=g, device='cuda')
    qe = torch.sigmoid(torch.randn(CK, q, generator=g, device='cuda'))
    mk = torch.cat([qk.repeat_interleave(near, 1) + 0.05 * torch.randn(CK, q * near, generator=g, device='cuda'),
                    torch.randn(CK, far, generator=g, device='cuda')], 1)
    perm = torch.randperm(mk.shape[1], generator=g, device='cuda')
    mk = mk[:, perm].contiguous()
    n = mk.shape[1]
    ms = 1 + torch.rand(n, generator=g, device='cuda')
    win = Window(nat, mk, ms, torch.randn(128, n, generator=g, device='cuda'), lead)
    sim = win.sim64(qk, qe)
    top = torch.sort(sim, 0, descending=True)[0]
    assert float((top[28] - top[29]).min()) > 1.0  # far beyond the bound's 1/512 + 1e-3 allowance
    packed = _pack_q(nat, qk, qe)
    outs = Outputs()
    cold, cold_w, _ = _topk(nat, win, packed, q, top_k, outs)
    torch.cuda.synchronize()
    _check_selection(cold, cold_w, sim, top_k, lead, 'warm-start bank')
    prev = cold.clone()
    r = torch.arange(q, device='cuda')
    a, b, c = r % 3 == 0, r % 3 == 1, r % 3 == 2
    prev[a, :top_k] = cold[a, :1]                              # the top slot repeated top_k times
    prev[b, top_k - 1] = cold[b, 0]                            # the last (30th) entry replaced by the first
    bad = torch.where(r % 2 == 0, win.nw + r % 50, r % lead).int()
    prev[c, 5] = bad[c]                                        # out of range: past the window or a lead slot
    warm, warm_w, thr = _topk(nat, win, packed, q, top_k, outs, prev=prev)
    ok, ok_w, ok_thr = _topk(nat, win, packed, q, top_k, outs, prev=cold.clone())
    torch.cuda.synchronize()
    outs.check_guards()
    for got, got_w, what in ((warm, warm_w, 'repeated / invalid'), (ok, ok_w, 'valid')):
        diff = (got != cold).any(1) | (got_w != cold_w).any(1)
        assert not bool(diff.any()), f'{what} prev_idx changed {int(diff.sum())} reads'
    assert bool((thr == float('-inf')).all()), 'a row with a repeated or invalid slot got a bound'
    assert bool(torch.isfinite(ok_thr).all())


# ------------------------------------------------------------------------------------------------- merge_lists
@gpu
@pytest.mark.parametrize('n_lists', [1, 4, 16])
@pytest.mark.parametrize('top_k', [1, 30, 32])
def test_merge_lists_matches_the_rule(n_lists, top_k):
    nat = _nat()
    rng = np.random.default_rng(n_lists * 100 + top_k)
    q, pitch = 301, 333
    vals = np.full((n_lists, LP, pitch), np.nan, np.float32)
    ids = np.full((n_lists, LP, pitch), -1, np.int32)
    for i in range(q):
        slots = rng.permutation(100000)[:n_lists * top_k].reshape(n_lists, top_k)  # lists hold disjoint slots
        v = np.round(rng.normal(size=(n_lists, top_k)), 1).astype(np.float32)     # coarse values: ties across lists
        v = -np.sort(-v, 1)
        keep = rng.random((n_lists, top_k)) < (0.02 if i % 5 == 0 else 0.9)      # empty entries; short rows
        keep[0, 0] = True
        ids[:, :top_k, i] = np.where(keep, slots, -1)
        vals[:, :top_k, i] = np.where(keep, v, np.where(rng.random((n_lists, top_k)) < 0.5, np.inf, np.nan))
    assert top_k == 1 or any((ids[:, :top_k, i] >= 0).sum() < top_k for i in range(q))
    outs = Outputs()
    oi, ow, os_ = outs.new((q, LP), torch.int32), outs.new((q, LP), torch.float32), outs.new((q, LP), torch.float32)
    nat.merge_lists(torch.from_numpy(vals).cuda(), torch.from_numpy(ids).cuda(), n_lists, top_k, q, pitch, oi, ow, os_)
    torch.cuda.synchronize()
    outs.check_guards()
    ri, rw, rs = merge_ref(vals, ids, top_k, q)
    assert np.array_equal(oi.cpu().numpy(), ri), 'merged indices differ from the rule'
    assert np.array_equal(os_.cpu().numpy(), rs)
    err = float(np.abs(ow.cpu().numpy().astype(np.float64) - rw).max())
    _report(f'merge lists={n_lists} k={top_k} weights', err, 1e-6)
    assert err < 1e-6


# ------------------------------------------------------------------------------------------------- scatter read-out
@gpu
@pytest.mark.parametrize('n_ranks', [3, 8])
@pytest.mark.parametrize('ld_pad', [0, 1])
def test_scatter_readout_to_local_buffers(n_ranks, ld_pad):
    """Each destination buffer receives (red.add into zero) exactly the plain sparse read-out of the groups it owns."""
    nat = _nat()
    g = _gen(n_ranks * 10 + ld_pad)
    slots, groups, cv, n, lead, q, top_k = 12, 11, 128, 3000, 4, 1000, 30
    mk, ms, qk, qe, mv = _keys(g, n, q, slots * cv)
    win = Window(nat, mk, ms, mv, lead, n_long=500)
    outs = Outputs()
    idx, w, _ = _topk(nat, win, _pack_q(nat, qk, qe), q, top_k, outs)
    # another rank's slots: weight 0 at slot 0, as the bank-sharded read localises its lists
    other = torch.rand(q, LP, generator=g, device='cuda') < 0.2
    idx = torch.where(other, torch.zeros_like(idx), idx).contiguous()
    w = torch.where(other, torch.zeros_like(w), w).contiguous()
    owner = [int(o) for o in torch.randint(0, n_ranks, (groups, ), generator=g, device='cuda')]
    val_row = [int(s) * cv for s in torch.randperm(slots, generator=g, device='cuda')[:groups]]
    ldo = q + ld_pad
    local, out_row = [0] * n_ranks, []
    for o in owner:
        out_row.append(local[o] * cv)
        local[o] += 1
    dst = [outs.new((max(1, k) * cv, ldo), torch.float32, torch.zeros(max(1, k) * cv * ldo, device='cuda'))
           for k in local]
    rws = torch.empty(nat.readout_sparse_workspace_bytes(q, win.nw), dtype=torch.uint8, device='cuda')
    nat.readout_sparse_scatter(win.vals(), win.cap, win.rows, val_row, out_row, owner, cv, idx, w, top_k, win.nw, q,
                               rws, [t.data_ptr() for t in dst], ldo)
    torch.cuda.synchronize()
    outs.check_guards()
    for r in range(n_ranks):
        mine = [i for i in range(groups) if owner[i] == r]
        if not mine:
            assert bool((dst[r] == 0).all())
            continue
        ref = outs.new((len(mine) * cv, ldo), torch.float32)
        nat.readout_sparse(win.vals(), win.cap, win.rows, [val_row[i] for i in mine], [out_row[i] for i in mine], cv,
                           idx, w, top_k, win.nw, q, rws, ref, ldo)
        torch.cuda.synchronize()
        assert torch.equal(dst[r][:, :q], ref[:, :q]), f'rank {r}: scattered read-out differs from the plain one'
        assert bool((dst[r][:, q:] == 0).all()), 'columns past q were written'
    _report(f'scatter ranks={n_ranks} ld_out={ldo}', 0.0, 0.0)


# ------------------------------------------------------------------------------------------------- bank data movement
@gpu
def test_bank_gathers_are_exact():
    nat = _nat()
    g = _gen(3)
    outs = Outputs()
    for row_bytes in (256, 512):
        src = torch.randint(-2 ** 31, 2 ** 31 - 1, (5000, row_bytes // 4), generator=g, device='cuda', dtype=torch.int32)
        idx = torch.randint(0, 5000, (3001, ), generator=g, device='cuda', dtype=torch.int32)
        idx[100:110] = idx[5]  # repeated indices
        dst = outs.new((3001, row_bytes // 4), torch.int32)
        nat.gather_rows(dst, src, idx, 3001, row_bytes)
        torch.cuda.synchronize()
        assert torch.equal(dst, src.index_select(0, idx.long()))
    src = torch.randn(9000, generator=g, device='cuda')
    idx = torch.randint(0, 9000, (4097, ), generator=g, device='cuda', dtype=torch.int32)
    dst = outs.new((4097, ), torch.float32)
    nat.gather_f32(dst, src, idx, 4097)
    # value columns: 16 objects x 512 channels, 40k gathered columns, ld != n on both sides
    rows, n, ld_src, ld_dst = 16 * 512, 40000, 41016, 40008
    src16 = torch.randn(rows, ld_src, generator=g, device='cuda').half()
    cols = torch.randint(0, ld_src, (n, ), generator=g, device='cuda', dtype=torch.int32)
    cols[:64] = cols[64]
    dst16 = outs.new((rows, ld_dst), torch.float16)
    nat.gather_cols_f16(dst16, ld_dst, src16, ld_src, cols, rows, n)
    torch.cuda.synchronize()
    outs.check_guards()
    assert torch.equal(dst, src.index_select(0, idx.long()))
    assert torch.equal(dst16[:, :n], src16.index_select(1, cols.long()))
    assert bool(torch.isnan(dst16[:, n:].float()).all()), 'gather_cols_f16 wrote past n columns'


@gpu
def test_bank_packing_and_appends():
    nat = _nat()
    g = _gen(4)
    n, pos, cap = 1000, 13, 1100
    outs = Outputs()
    # token-major key rows with selection (the NHWC engine's append; prepend_long passes key rows the same way)
    key = torch.randn(n, CK, generator=g, device='cuda')
    sel = torch.sigmoid(torch.randn(n, CK, generator=g, device='cuda'))
    shr = 1 + torch.rand(n, generator=g, device='cuda')
    k_hi, k_lo = outs.new((cap, 2 * CK), torch.float16), outs.new((cap, 2 * CK), torch.float16)
    neg_s, raw_shr = outs.new((cap, ), torch.float32), outs.new((cap, ), torch.float32)
    raw_key, raw_sel = outs.new((cap, CK), torch.float32), outs.new((cap, CK), torch.float32)
    nat.pack_keys(key, sel, 1, CK, shr, CK, n, k_hi[pos:], k_lo[pos:], neg_s[pos:], raw_key[pos:], raw_sel[pos:],
                  raw_shr[pos:])
    # values: fp32 channel-major and fp16 token-major appends at an unaligned window offset
    cv = 512
    vsrc = torch.randn(cv, n, generator=g, device='cuda')
    vtok = torch.randn(n, cv, generator=g, device='cuda').half()
    va, vt = outs.new((cv, cap), torch.float16), outs.new((cv, cap), torch.float16)
    nat.append_values(vsrc, n, va[:, pos:], cap, cv, n)
    nat.transpose_append(vtok, vt[:, pos:], cap, n, cv)
    torch.cuda.synchronize()
    outs.check_guards()
    w = slice(pos, pos + n)
    s = shr.double() / 8
    want = torch.cat([s[:, None] * key.double() ** 2, s[:, None] * key.double()], 1)
    got = k_hi[w].double() + k_lo[w].double()
    # s = shrinkage * rsqrtf(64): rsqrtf's 2 ulp (4 * 2^-24 relative) plus one rounding; times k twice, one rounding
    # each: 7 * 2^-24.  The fp16 lo part of the split rounds the residual |x - hi| <= 2^-11 |x| by 2^-11 of it
    # (4 * 2^-24 relative), or by 2^-25 absolute where lo is fp16-subnormal.  Total 11 * 2^-24 < 2^-20.
    err = (got - want).abs()
    bound = 2.0 ** -20 * want.abs() + 2.0 ** -25
    _report('pack_keys hi + lo (err / bound)', float((err / bound).max()), 1.0)
    assert bool((err <= bound).all())
    assert torch.equal(raw_key[w], key) and torch.equal(raw_sel[w], sel) and torch.equal(raw_shr[w], shr)
    assert float(((neg_s[w].double() + s) / s).abs().max()) <= 5 * 2.0 ** -24
    for buf in (k_hi, k_lo, raw_key, raw_sel):
        assert bool(torch.isnan(buf[:pos].float()).all()) and bool(torch.isnan(buf[pos + n:].float()).all())
    assert torch.equal(va[:, w], vsrc.half()) and torch.equal(vt[:, w], vtok.t())
    for buf in (va, vt):
        assert bool(torch.isnan(buf[:, :pos].float()).all()) and bool(torch.isnan(buf[:, pos + n:].float()).all())


# ------------------------------------------------------------------------------------------------- product path
@gpu
def test_fused_and_dense_read_paths_are_identical():
    """The memory manager's event stream (appends, consolidation, eviction, a second bucket, a purge) read through the
    fused sparse read-out and through the dense-affinity GEMM: every read is bit-identical."""
    from deva.inference.memory_manager import MemoryManager
    _nat()
    cfg = dict(key_dim=64, value_dim=128, pix_feat_dim=512, mem_every=1, enable_long_term=True, chunk_size=-1, top_k=30,
               enable_long_term_count_usage=True, max_mid_term_frames=6, min_mid_term_frames=3, num_prototypes=128,
               max_long_term_elements=300)
    g = torch.Generator().manual_seed(4)
    fused, dense = MemoryManager(cfg), MemoryManager(cfg)
    fused.fused_min_work, dense.fused_min_work = 0, 1 << 62
    fused.readout_layout = dense.readout_layout = 'nchw'  # compare the fp32 reads, not their fp16 roundings
    objs = [3, 9]
    h, w = 6, 8
    for t in range(26):
        if t == 7:
            objs = objs + [21]
        if t == 15:
            objs = [3, 21]
            fused.purge_except(objs)
            dense.purge_except(objs)
        key = torch.randn(1, 64, h, w, generator=g).cuda()
        shr = (1 + 0.05 * torch.rand(1, 1, h, w, generator=g)).cuda()
        sel = torch.sigmoid(torch.randn(1, 64, h, w, generator=g)).cuda()
        val = torch.randn(1, len(objs), 128, h, w, generator=g).cuda()
        if t > 0:
            a, b = fused.match_memory(key, sel), dense.match_memory(key, sel)
            assert a.keys() == b.keys()
            for o in a:
                assert torch.equal(a[o], b[o]), f'step {t}, object {o}: fused and dense reads differ'
        fused.add_memory(key, shr, val, list(objs), selection=sel)
        dense.add_memory(key, shr, val, list(objs), selection=sel)
    for b in fused._banks:  # usage is accumulated with float atomics, in no fixed order
        torch.testing.assert_close(fused._banks[b].use_cnt, dense._banks[b].use_cnt, rtol=1e-5, atol=1e-6)
