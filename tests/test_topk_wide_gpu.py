"""Memory reads at top_k beyond the 32-entry running lists of sim_topk: the wide selection kernel (csrc/simtopk.cu), the
sparse read-outs at a wider list pitch (csrc/readout.cu), MemoryManager's wide path, the sharded core's wide merge, and
DEVAInferenceCore.step at top_k 50 and 100 against the reference-minted fixture tests/golden/topk_wide.

Kernel-level checks are against float64 (oracle/memory_math.py) with the bounds of tests/test_memory_kernels_gpu.py:
the selected set must be exact wherever the gap between the k-th and the (k+1)-th float64 similarity exceeds twice the
similarity bound, and the weights, similarities and usage must be within their bounds over the slots the kernel chose.
"""
import json
import os
import socket
import sys
import time
from datetime import timedelta

import numpy as np
import pytest
import torch
import torch.distributed as dist

from oracle import memory_math as mm


def gpu(fn):
    """Needs a CUDA device: selected by ``-m gpu``, skipped (not failed) where there is none."""
    return pytest.mark.gpu(pytest.mark.skipif(not torch.cuda.is_available(), reason='needs a CUDA device')(fn))


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CK, CV = 64, 128
SIM_ABS = 1e-4        # similarity bound of tests/test_memory_kernels_gpu.py
W_ABS = 2e-5          # softmax weight bound of the memory-read tests
USE_REL = 1e-4        # usage: fp32 atomic sums of up to 8160 weights per slot, relative to max(1, max |usage|)
READ_REL = 1e-3       # read-out bound, relative to max(1, max |reference|) (tests/test_sharded_ranks_gpu.py)
PROB_TOL = 1e-3       # |prob - reference| budget of tests/test_step_gpu.py, on every frame whose reads select the
                      # float64 top-k set for every query
PROB_NEAR_TIE = 5e-3  # ... and on a frame where a query's k-th and (k+1)-th slots are closer than the similarity error
                      # of fp32 (the kernel's or the reference's), so that either may be selected: one such query at
                      # top_k 50, frame 9 (gap 6.2e-7) moves that frame to 2.8e-3 (H100 80GB HBM3, 700 W)
PROB_CLIP = 2e-3      # |prob - plain core| of a sharded session (tests/test_sharded_ranks_gpu.py)


def _nat():
    from deva import _native
    _native.require_device()
    return _native


def _report(name, err, bound):
    print(f'[topk-wide] {name}: measured {err:.3e}, bound {bound:.3e}')


class Bank:
    """n memory slots behind `lead` alignment slots whose key rows are NaN (the kernels must never read them)."""

    def __init__(self, nat, mk, ms, lead):
        n = mk.shape[1]
        self.n, self.lead, self.nw = n, lead, lead + n
        self.k_hi = torch.full((self.nw, 2 * CK), float('nan'), dtype=torch.float16, device='cuda')
        self.k_lo = torch.full_like(self.k_hi, float('nan'))
        self.neg_s = torch.full((self.nw, ), float('nan'), device='cuda')
        raw_key, raw_shr = torch.empty(n, CK, device='cuda'), torch.empty(n, device='cuda')
        nat.pack_keys(mk.contiguous(), None, n, 1, ms.contiguous(), CK, n, self.k_hi[lead:], self.k_lo[lead:],
                      self.neg_s[lead:], raw_key, None, raw_shr)
        self.mk, self.ms = mk, ms


def _query(nat, qk, qe):
    q = qk.shape[1]
    q_hi = torch.empty(q, 2 * CK, dtype=torch.float16, device='cuda')
    q_lo, bsq = torch.empty_like(q_hi), torch.empty(q, device='cuda')
    nat.pack_query(qk.contiguous(), qe.contiguous(), q, 1, CK, q, q_hi, q_lo, bsq)
    return q_hi, q_lo, bsq


def _inputs(seed, n, q):
    g = torch.Generator(device='cuda').manual_seed(seed)
    mk = torch.randn(CK, n, generator=g, device='cuda')
    ms = 1 + torch.rand(n, generator=g, device='cuda')
    qk = torch.randn(CK, q, generator=g, device='cuda')
    qe = torch.sigmoid(torch.randn(CK, q, generator=g, device='cuda'))
    return mk, ms, qk, qe


def _wide(nat, bank, qry, top_k, ld=None, aff=False, use=None, life=None, n_long=0, count_long=False, count_work=False):
    q = qry[0].shape[0]
    ld = ld or nat.list_pitch(top_k)
    ws = torch.empty(nat.sim_topk_wide_workspace_bytes(q, bank.nw), dtype=torch.uint8, device='cuda')
    idx = torch.full((q, ld), -7, dtype=torch.int32, device='cuda')
    w, sim = torch.full((q, ld), float('nan'), device='cuda'), torch.full((q, ld), float('nan'), device='cuda')
    ldp = (bank.nw + 7) // 8 * 8
    P = torch.full((q, ldp), float('nan'), dtype=torch.float16, device='cuda') if aff else None
    nat.sim_topk_wide(bank.k_hi, bank.k_lo, bank.neg_s, bank.nw, bank.lead, *qry, q, CK, top_k, ws, idx, w, ld, P,
                      ldp if aff else 0, use, life, n_long, count_long, count_work, out_sim=sim)
    return idx, w, sim, P


def _check_selection(name, bank, qk, qe, top_k, idx, w, sim):
    """Exact set where the float64 gap allows it, ascending slot order, padding, weights and similarities in bound."""
    q = qk.shape[1]
    s64 = mm.similarity(bank.mk.double(), bank.ms.double(), qk.double(), qe.double())  # [n, q]
    sel = idx[:, :top_k].long() - bank.lead                                          # [q, k] memory slot
    assert bool((sel >= 0).all() and (sel < bank.n).all()), f'{name}: slot outside the window'
    if top_k > 1:
        assert bool((sel[:, 1:] > sel[:, :-1]).all()), f'{name}: entries not in ascending slot order'
    ld = idx.shape[1]
    if ld > top_k:
        assert bool((idx[:, top_k:] == 0).all() and (w[:, top_k:] == 0).all()), f'{name}: padding'
        assert bool(torch.isinf(sim[:, top_k:]).all() and (sim[:, top_k:] < 0).all()), f'{name}: padding similarity'
    vals, ref = torch.topk(s64, top_k + (1 if top_k < bank.n else 0), dim=0)
    gap = (vals[top_k - 1] - vals[top_k]) if top_k < bank.n else torch.full((q, ), float('inf'), device='cuda',
                                                                            dtype=torch.float64)
    clear = gap > 2 * SIM_ABS
    same = (ref[:top_k].t().sort(1)[0] == sel.sort(1)[0]).all(1)
    bad = int((clear & ~same).sum())
    assert bad == 0, f'{name}: {bad} queries with a clear k-th gap select another set'
    s_sel = s64.t().gather(1, sel)                                                     # [q, k]
    w64 = torch.softmax(s_sel, dim=1)
    e_sim = float((sim[:, :top_k].double() - s_sel).abs().max())
    e_w = float((w[:, :top_k].double() - w64).abs().max())
    _report(f'{name} similarity ({int(clear.sum())}/{q} queries with a clear gap)', e_sim, SIM_ABS)
    _report(f'{name} weights', e_w, W_ABS)
    assert e_sim <= SIM_ABS and e_w <= W_ABS
    return sel


# c2 / c3 read shapes of the benchmark (ragged: Q and N are no multiple of the tiles), each with its k = every slot
SHAPES = {'c2': (1620, 2000, 3, 700), 'c3': (8160, 10000, 5, 2500)}   # q, n, lead, long-term slots


@gpu
@pytest.mark.parametrize('shape', sorted(SHAPES))
def test_wide_selection_matches_float64(shape):
    nat = _nat()
    q, n, lead, n_long = SHAPES[shape]
    mk, ms, qk, qe = _inputs(1 if shape == 'c2' else 2, n, q)
    bank = Bank(nat, mk, ms, lead)
    qry = _query(nat, qk, qe)
    count_long = shape == 'c2'   # c2 counts both regions, c3 only the working memory
    for top_k in (33, 48, 64, 100, 128, 256, 1000, n):
        use = torch.zeros(bank.nw, device='cuda')
        life = torch.zeros(bank.nw, device='cuda')
        idx, w, sim, _ = _wide(nat, bank, qry, top_k, use=use, life=life, n_long=lead + n_long, count_long=count_long,
                               count_work=True)
        sel = _check_selection(f'{shape} top_k {top_k}', bank, qk, qe, top_k, idx, w, sim)
        want = torch.zeros(bank.nw, dtype=torch.float64, device='cuda')
        want.index_add_(0, (sel + lead).reshape(-1), w[:, :top_k].double().reshape(-1))
        lo = lead if count_long else lead + n_long
        want[:lo] = 0
        err = float((use.double() - want).abs().max()) / max(1.0, float(want.abs().max()))
        _report(f'{shape} top_k {top_k} usage (relative)', err, USE_REL)
        assert err <= USE_REL
        tick = torch.zeros(bank.nw, device='cuda')
        tick[lo:] = 1
        assert torch.equal(life, tick), f'{shape} top_k {top_k}: life ticks'


@gpu
def test_wide_selection_streams_long_rows():
    """A window of more than 50 000 slots: the rows do not fit in shared memory and every radix pass re-reads them."""
    nat = _nat()
    q, n, lead = 517, 52_003, 6
    mk, ms, qk, qe = _inputs(3, n, q)
    bank = Bank(nat, mk, ms, lead)
    qry = _query(nat, qk, qe)
    for top_k in (33, 100, 1000):
        idx, w, sim, _ = _wide(nat, bank, qry, top_k)
        _check_selection(f'streamed n {n} top_k {top_k}', bank, qk, qe, top_k, idx, w, sim)


def _fp32_sims(nat, bank, qry):
    """The kernel's own fp32 similarities of every slot [q, n] (sim_dense_softmax runs the same GEMM)."""
    q = qry[0].shape[0]
    ld = (bank.nw + 7) // 8 * 8
    sim_ws = torch.empty(q, ld, device='cuda')
    aff = torch.zeros(q, ld, dtype=torch.float16, device='cuda')
    nat.sim_dense_softmax(bank.k_hi, bank.k_lo, bank.neg_s, None, bank.nw, bank.lead, *qry, q, CK, sim_ws, ld, aff, ld,
                          None)
    return sim_ws[:, bank.lead:bank.nw]


@gpu
def test_exact_ties_follow_the_tie_rule():
    """Slots i and i + 48 k hold the same key and shrinkage, so their similarities are bit-identical: at the threshold
    the lower slots win, as in sim_topk.  At top_k 32 the wide path selects exactly what sim_topk selects."""
    nat = _nat()
    q, base, copies, lead = 300, 48, 13, 2
    mk, ms, qk, qe = _inputs(4, base, q)
    mk, ms = mk.repeat(1, copies), ms.repeat(copies)
    bank = Bank(nat, mk, ms, lead)
    qry = _query(nat, qk, qe)
    s32 = _fp32_sims(nat, bank, qry)                                       # [q, n]
    for top_k in (32, 40, 100, 333):
        idx, w, sim, _ = _wide(nat, bank, qry, top_k)
        # rank by (similarity desc, slot asc): a stable sort by slot, then by similarity
        order = torch.sort(s32, dim=1, descending=True, stable=True)[1]
        want = order[:, :top_k].sort(1)[0] + lead
        assert torch.equal(idx[:, :top_k].long(), want), f'top_k {top_k}: tie rule'
        kth = s32.gather(1, order[:, top_k - 1:top_k])
        ties = int(((s32 == kth).sum(1) > 1).sum())
        print(f'[topk-wide] ties top_k {top_k}: {ties}/{q} queries have several slots at the threshold value')
        assert ties > 0
        assert torch.equal(sim[:, :top_k], s32.gather(1, idx[:, :top_k].long() - lead))
        if top_k == 32:
            ws = torch.empty(nat.simtopk_workspace_bytes(q), dtype=torch.uint8, device='cuda')
            n_idx = torch.empty(q, 32, dtype=torch.int32, device='cuda')
            n_w = torch.empty(q, 32, device='cuda')
            nat.sim_topk(bank.k_hi, bank.k_lo, bank.neg_s, bank.nw, lead, *qry, q, CK, 32, ws, n_idx, n_w, None, 0,
                         None, None, 0, False, False)
            srt, perm = n_idx.sort(1)
            assert torch.equal(srt, idx), 'top_k 32: the wide path selects another set than sim_topk'
            ulp = float(((n_w.gather(1, perm) - w).abs() / (w.abs() * 2.0 ** -23 + 1e-30)).max())
            _report('top_k 32 weights wide vs sim_topk, in ulps', ulp, 8)
            assert ulp <= 8


def _merge_ref(vals, ids, top_k):
    """vals/ids [L, ld, q] numpy -> per query the selected (list, entry) positions in input order and their values."""
    L, ld, q = vals.shape
    out = []
    for j in range(q):
        v, i = vals[:, :, j].reshape(-1), ids[:, :, j].reshape(-1)
        ok = np.nonzero(i >= 0)[0]
        rank = sorted(ok, key=lambda c: (-float(v[c]), int(i[c])))[:top_k]
        out.append(sorted(rank))
    return out


@gpu
@pytest.mark.parametrize('n_lists,ld,top_k,k_loc', [(2, 64, 64, 64), (3, 64, 50, 40), (5, 128, 100, 100),
                                                    (16, 256, 200, 17), (2, 64, 64, 20)])
def test_merge_lists_wide_follows_the_rule(n_lists, ld, top_k, k_loc):
    """n candidate lists with explicit slot ids (distinct per query), empty entries (id -1) and k_loc < top_k; values
    quantised to 1/4 so that ties at the threshold are common.  Where the lists hold fewer than top_k candidates all are
    taken and the rest of the row is empty."""
    nat = _nat()
    q = 203
    g = np.random.default_rng(n_lists * 1000 + top_k)
    vals = np.round(g.normal(size=(n_lists, ld, q)) * 4) / 4
    ids = np.stack([g.permutation(n_lists * ld * 4)[:n_lists * ld].reshape(n_lists, ld) for _ in range(q)], axis=-1)
    ids[:, k_loc:, :] = -1
    ids[g.random(ids.shape) < 0.05] = -1
    vals[ids < 0] = -np.inf
    pv = torch.tensor(vals, dtype=torch.float32, device='cuda')
    pi = torch.tensor(ids, dtype=torch.int32, device='cuda')
    o_idx = torch.full((q, ld), -7, dtype=torch.int32, device='cuda')
    o_w, o_sim = torch.full((q, ld), float('nan'), device='cuda'), torch.full((q, ld), float('nan'), device='cuda')
    nat.merge_lists_wide(pv, pi, n_lists, ld, top_k, q, q, o_idx, o_w, o_sim)
    got_i, got_w, got_s = o_idx.cpu().numpy(), o_w.cpu().numpy(), o_sim.cpu().numpy()
    worst = 0.0
    for j, pos in enumerate(_merge_ref(vals, ids, top_k)):
        k = len(pos)
        flat_i, flat_v = ids[:, :, j].reshape(-1), vals[:, :, j].reshape(-1)
        assert got_i[j, :k].tolist() == flat_i[pos].tolist(), f'query {j}: selection or order'
        assert np.array_equal(got_s[j, :k], flat_v[pos].astype(np.float32))
        e = np.exp(flat_v[pos] - flat_v[pos].max())
        worst = max(worst, float(np.abs(got_w[j, :k] - e / e.sum()).max()))
        assert (got_i[j, k:] == 0).all() and (got_w[j, k:] == 0).all() and np.isneginf(got_s[j, k:]).all()
    _report(f'merge {n_lists} lists of {ld}, top_k {top_k}: weights', worst, 1e-6)
    assert worst <= 1e-6


@gpu
@pytest.mark.parametrize('pitch', [64, 256])
def test_sparse_and_dense_readouts_agree_at_wide_pitch(pitch):
    nat = _nat()
    q, n, lead, objs = 1100, 3000, 3, 3
    mk, ms, qk, qe = _inputs(5 + pitch, n, q)
    bank = Bank(nat, mk, ms, lead)
    qry = _query(nat, qk, qe)
    g = torch.Generator(device='cuda').manual_seed(pitch)
    rows = objs * CV
    mv = torch.randn(rows, n, generator=g, device='cuda')
    ld_v = (bank.nw + 7) // 8 * 8
    values = torch.zeros(rows, ld_v, dtype=torch.float16, device='cuda')
    nat.append_values(mv, n, values[:, lead:], ld_v, rows, n)
    for top_k in (pitch - 31, pitch):
        idx, w, _, P = _wide(nat, bank, qry, top_k, ld=pitch, aff=True)
        ldp = P.shape[1]
        rws = torch.empty(nat.readout_sparse_wide_workspace_bytes(q, bank.nw, pitch), dtype=torch.uint8, device='cuda')
        sparse = torch.full((rows, q), float('nan'), device='cuda')
        dense = torch.full((rows, q), float('nan'), device='cuda')
        rv = [o * CV for o in range(objs)]
        ro = [(objs - 1 - o) * CV for o in range(objs)]   # objects written in reverse order
        nat.readout_sparse_wide(values, ld_v, rows, rv, ro, CV, idx, w, pitch, top_k, bank.nw, q, rws, sparse, q)
        nat.readout(values, ld_v, rows, rv, ro, CV, P, ldp, bank.nw, q, dense, q)
        aff = torch.zeros(q, bank.nw, dtype=torch.float64, device='cuda')
        aff.scatter_(1, idx[:, :top_k].long(), w[:, :top_k].double())
        ref = mm.readout(aff[:, lead:].t(), values[:, lead:bank.nw].double())    # [rows, q]
        ref = torch.cat([ref[(objs - 1 - o) * CV:(objs - o) * CV] for o in range(objs)])
        scale = max(1.0, float(ref.abs().max()))
        e_s = float((sparse.double() - ref).abs().max()) / scale
        e_d = float((dense.double() - ref).abs().max()) / scale
        e_sd = float((sparse - dense).abs().max()) / scale
        _report(f'pitch {pitch} top_k {top_k} sparse / dense / sparse-dense read-out (relative)', max(e_s, e_d, e_sd),
                READ_REL)
        assert max(e_s, e_d, e_sd) <= READ_REL


@gpu
def test_errors_raise():
    nat = _nat()
    q, n, lead = 100, 200, 2
    mk, ms, qk, qe = _inputs(6, n, q)
    bank = Bank(nat, mk, ms, lead)
    qry = _query(nat, qk, qe)
    for top_k in (0, -3, n + 1):
        with pytest.raises(RuntimeError):
            _wide(nat, bank, qry, top_k, ld=256)
    with pytest.raises(RuntimeError, match='ld_list'):
        _wide(nat, bank, qry, 40, ld=40)
    _wide(nat, bank, qry, n)  # every slot
    pv = torch.zeros(2, 64, q, device='cuda')
    pi = torch.zeros(2, 64, q, dtype=torch.int32, device='cuda')
    out_i, out_w = torch.empty(q, 64, dtype=torch.int32, device='cuda'), torch.empty(q, 64, device='cuda')
    for top_k in (0, 65):
        with pytest.raises(RuntimeError):
            nat.merge_lists_wide(pv, pi, 2, 64, top_k, q, q, out_i, out_w)


# ------------------------------------------------------------------------------------------------- memory manager
def _manager(top_k, use_long=True):
    from deva.inference.memory_manager import MemoryManager
    cfg = dict(key_dim=CK, value_dim=512, pix_feat_dim=512, mem_every=1, enable_long_term=use_long, chunk_size=-1,
               top_k=top_k, enable_long_term_count_usage=True, max_mid_term_frames=10, min_mid_term_frames=5,
               num_prototypes=128, max_long_term_elements=10000)
    return MemoryManager(cfg)


def _fill(mm_, seed, h, w, frames, k=2):
    g = torch.Generator(device='cuda').manual_seed(seed)
    for _ in range(frames):
        key = torch.randn(1, CK, h, w, generator=g, device='cuda')
        shr = 1 + torch.rand(1, 1, h, w, generator=g, device='cuda')
        sel = torch.sigmoid(torch.randn(1, CK, h, w, generator=g, device='cuda'))
        val = torch.randn(1, k, CV, h, w, generator=g, device='cuda')
        mm_.add_memory(key, shr, val, list(range(1, k + 1)), selection=sel)
    qk = torch.randn(1, CK, h, w, generator=g, device='cuda')
    qe = torch.sigmoid(torch.randn(1, CK, h, w, generator=g, device='cuda'))
    return qk, qe


class _Counting:
    def __init__(self, nat, names):
        self.nat, self.calls, self.saved = nat, {n: 0 for n in names}, {}
        for name in names:
            fn = getattr(nat, name)
            self.saved[name] = fn

            def wrap(*a, _fn=fn, _name=name, **k):
                self.calls[_name] += 1
                return _fn(*a, **k)
            setattr(nat, name, wrap)

    def restore(self):
        for name, fn in self.saved.items():
            setattr(self.nat, name, fn)


@gpu
@pytest.mark.parametrize('fused_min_work', [16_000_000, 0])
def test_narrow_reads_keep_the_existing_path(fused_min_work):
    """top_k 30 calls only the existing entry points, twice (warm start on the second read), and gives the same
    read-out as before; top_k 50 calls only the wide ones and matches float64 of the whole read."""
    nat = _nat()
    names = ['sim_topk', 'readout_sparse', 'readout', 'sim_topk_wide', 'readout_sparse_wide']
    h, w = 30, 54
    for top_k in (30, 50):
        mgr = _manager(top_k)
        mgr.readout_layout = 'nchw'
        mgr.fused_min_work = fused_min_work
        qk, qe = _fill(mgr, 7, h, w, 3)
        count = _Counting(nat, names)
        try:
            a = mgr.match_memory(qk, qe)
            b = mgr.match_memory(qk, qe)
        finally:
            count.restore()
        wide = top_k > 30
        narrow_calls = count.calls['sim_topk'] + count.calls['readout_sparse']
        wide_calls = count.calls['sim_topk_wide'] + count.calls['readout_sparse_wide']
        assert (wide_calls == 0) != wide and (narrow_calls == 0) == wide, count.calls
        assert count.calls['sim_topk' + ('_wide' if wide else '')] == 2
        for o in a:
            assert torch.equal(a[o], b[o]), 'a repeated read differs'
        bank = next(iter(mgr._banks.values()))
        w0, lead, n_window = bank.window()
        n = n_window - lead
        key = bank.raw_key[w0 + lead:w0 + n_window].t().double()
        shr = bank.raw_shr[w0 + lead:w0 + n_window].double()
        vals = bank.values[:, :, w0 + lead:w0 + n_window].double().reshape(-1, n)
        ref, _, _, _ = mm.read(key, shr, qk[0].reshape(CK, -1).double(), qe[0].reshape(CK, -1).double(), vals, top_k)
        got = torch.cat([a[o].reshape(CV, -1) for o in sorted(a)]).double()
        err = float((got - ref).abs().max()) / max(1.0, float(ref.abs().max()))
        _report(f'match_memory top_k {top_k} (fused_min_work {fused_min_work}) vs float64', err, READ_REL)
        assert err <= READ_REL


@gpu
def test_manager_top_k_above_the_window_raises():
    mgr = _manager(1000)
    qk, qe = _fill(mgr, 8, 10, 12, 2)
    with pytest.raises(RuntimeError, match='exceeds'):
        mgr.match_memory(qk, qe)


# ------------------------------------------------------------------------------------------------- end to end
def _topk_clip(golden_dir):
    g = {k: torch.from_numpy(v) for k, v in np.load(os.path.join(golden_dir, 'topk_wide.npz')).items()}
    meta = json.load(open(os.path.join(golden_dir, 'topk_wide.json')))
    gen = torch.Generator().manual_seed(11)      # tests/golden/make_topk_golden.py:clip()
    H, W, T = 160, 192, 16
    base = torch.randn(3, H, W, generator=gen)
    frames = torch.stack([base + 0.2 * torch.randn(3, H, W, generator=gen) for _ in range(T)])
    assert abs(float(frames.double().sum()) - meta['frames_sum']) < 1e-6 * meta['frames_abs_sum']
    assert abs(float(frames.double().abs().sum()) - meta['frames_abs_sum']) < 1e-9 * meta['frames_abs_sum']
    g['frames'] = frames
    return g, meta


def _run_topk_clip(core, g, dev, reads=None):
    """reads (optional): a list that receives one list per frame, filled by a wrapper of the core's memory read."""
    T = g['frames'].shape[0]
    out = dict(probs=[], sizes=[], ids=[])
    for t in range(T):
        if reads is not None:
            reads.append([])
        img = g['frames'][t].to(dev)
        if t == 0:
            p = core.step(img, g['mask0'].long().to(dev), [1, 2])
        elif t == 6:
            p = core.step(img, g['mask6'].long().to(dev), [7])
        else:
            p = core.step(img, end=(t == T - 1))
        out['probs'].append(p.float().cpu())
        mem = core.memory
        out['sizes'].append({str(b): [mem.work_mem.size(b), mem.long_mem.size(b)] for b in mem.work_mem.buckets})
        out['ids'].append(core.object_manager.tmp_to_obj_cls(p.argmax(0)).cpu())
    return out


def _net(cfg, dev):
    from deva.model.network import DEVA
    from deva.model.param_spec import synthetic_state_dict
    net = DEVA(cfg).to(dev).eval()
    net.load_weights({k: v.to(dev) for k, v in synthetic_state_dict(seed=1).items()})
    return net


def _audit_reads(mgr, top_k, log):
    """Wrap mgr.match_memory: before every read, select each bank's top_k with sim_topk_wide on the read's own operands
    and compare with float64.  log[-1] receives, per bank, the float64 k-th gaps of the queries whose set differs."""
    nat = _nat()
    read = mgr.match_memory

    def audited(query_key, selection):
        qk = mgr._ck_n(query_key[0]).contiguous()
        qe = mgr._ck_n(selection[0]).contiguous()
        q = qk.shape[1]
        qry = _query(nat, qk, qe)
        for bank in mgr._banks.values():
            w0, lead, nw = bank.window()
            n, k = nw - lead, min(top_k, nw - lead)
            win = Bank.__new__(Bank)
            win.n, win.lead, win.nw = n, lead, nw
            win.k_hi, win.k_lo, win.neg_s = bank.k_hi[w0:], bank.k_lo[w0:], bank.neg_s[w0:]
            idx, _, _, _ = _wide(nat, win, qry, k)
            sel = idx[:, :k].long() - lead
            s64 = mm.similarity(bank.raw_key[w0 + lead:w0 + nw].t().double(), bank.raw_shr[w0 + lead:w0 + nw].double(),
                                qk.double(), qe.double())
            vals, ref = torch.topk(s64, min(k + 1, n), dim=0)
            differ = (ref[:k].t().sort(1)[0] != sel.sort(1)[0]).any(1)
            gaps = (vals[k - 1] - vals[k])[differ].tolist() if k < n else []
            assert len(gaps) == int(differ.sum())
            log[-1].append(gaps)
        return read(query_key, selection)
    mgr.match_memory = audited


@gpu
@pytest.mark.parametrize('top_k', [50, 100])
def test_step_matches_reference_at_wide_top_k(top_k, golden_dir):
    """The clip against the reference: bank sizes and confident ids exact on every frame; probabilities within 1e-3 on
    every frame whose reads select the float64 top-k set.  A query whose k-th and (k+1)-th float64 similarities are
    closer than fp32 can resolve may select either slot, here and in the reference; such a frame gets PROB_NEAR_TIE."""
    from deva.inference.inference_core import DEVAInferenceCore
    _nat()
    g, meta = _topk_clip(golden_dir)
    cfg = meta['configs'][str(top_k)]
    np.random.seed(42)
    core = DEVAInferenceCore(_net(cfg, 'cuda'), cfg)
    log = []
    _audit_reads(core.memory, top_k, log)
    run = _run_topk_clip(core, g, 'cuda', reads=log)
    near_tie = []
    for t, banks in enumerate(log):
        gaps = [x for b in banks for x in b]
        assert all(x < 2 * SIM_ABS for x in gaps), f'frame {t}: a query with a clear k-th gap selects another set'
        near_tie.append(bool(gaps))
        if gaps:
            print(f'[topk-wide] step top_k {top_k} frame {t}: {len(gaps)} queries at a near tie, float64 gaps',
                  ' '.join(f'{x:.1e}' for x in gaps))
    errs = []
    for t, p in enumerate(run['probs']):
        ref = g[f'k{top_k}_prob_{t:02d}']
        lattice = p[:, 1::4, 2::4]
        assert lattice.shape == ref.shape, t
        errs.append(float((lattice - ref).abs().max()))
        assert run['sizes'][t] == meta['sizes'][str(top_k)][t], (t, run['sizes'][t])
        confident = torch.from_numpy(np.unpackbits(g[f'k{top_k}_confident_{t:02d}'].numpy())[:p[0].numel()].astype(bool))
        got_ids = run['ids'][t].reshape(-1)[confident].to(torch.uint8)
        assert torch.equal(got_ids, g[f'k{top_k}_ids_{t:02d}'].reshape(-1)[confident]), f'frame {t}: confident ids'
    print(f'[topk-wide] step top_k {top_k} per frame:', ' '.join(f'{e:.2e}' for e in errs))
    exact = [e for e, nt in zip(errs, near_tie) if not nt]
    tied = [e for e, nt in zip(errs, near_tie) if nt]
    _report(f'step top_k {top_k} max |prob - reference| on {len(exact)} frames with exact selections', max(exact),
            PROB_TOL)
    if tied:
        _report(f'step top_k {top_k} max |prob - reference| on {len(tied)} frames with a near tie', max(tied),
                PROB_NEAR_TIE)
    assert max(exact) < PROB_TOL and max(tied, default=0.0) < PROB_NEAR_TIE


@gpu
def test_consensus_alignment_at_top_k_64(golden_dir):
    """spatial_alignment (a throw-away MemoryManager read) at top_k 64 runs through the wide path: a probability map
    that sums to one and differs from the same alignment at top_k 30."""
    from deva.inference.consensus_associated import spatial_alignment
    from deva.inference.image_feature_store import ImageFeatureStore
    _nat()
    g, meta = _topk_clip(golden_dir)
    cfg = dict(meta['configs']['50'], top_k=64)
    net = _net(cfg, 'cuda')
    store = ImageFeatureStore(net, no_warning=True)
    img0, img1 = g['frames'][0].cuda(), g['frames'][3].cuda()
    m = torch.stack([g['mask0'] == 1, g['mask0'] == 2]).float().cuda()
    prob64 = spatial_alignment(0, img0, m, 3, img1, net, store, cfg)[0]
    prob30 = spatial_alignment(0, img0, m, 3, img1, net, store, dict(cfg, top_k=30))[0]
    assert prob64.shape == prob30.shape == (3, 160, 192)
    assert float((prob64.float().sum(0) - 1).abs().max()) < 1e-4
    diff = float((prob64.float() - prob30.float()).abs().max())
    print(f'[topk-wide] spatial_alignment top_k 64 vs 30: max |prob difference| {diff:.3e}')
    assert diff > 0, 'top_k 64 read the memory exactly as top_k 30 did'


# ------------------------------------------------------------------------------------------------- sharded ranks
# The harness of tests/test_sharded_ranks_gpu.py: ranks as processes on one GPU, the tensor collectives staged through
# gloo on the host, peer memory mapped through CUDA IPC for real.
class StagedCollectives:
    def __getattr__(self, name):
        return getattr(dist, name)

    @staticmethod
    def all_gather_into_tensor(out, t, group=None):
        host = torch.empty(out.shape, dtype=out.dtype)
        dist.all_gather(list(host.unbind(0)), t.cpu().contiguous(), group=group)
        out.copy_(host)

    @staticmethod
    def all_reduce(t, op=dist.ReduceOp.SUM, group=None):
        host = t.cpu()
        dist.all_reduce(host, op=op, group=group)
        t.copy_(host)

    @staticmethod
    def all_to_all_single(out, t, group=None):
        host = torch.empty(out.shape, dtype=out.dtype)
        dist.all_to_all_single(host, t.cpu().contiguous(), group=group)
        out.copy_(host)


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


SHARD_TOP_K = 64
READER_Q, READER_N = 700, 2003


def _reader_inputs():
    g = torch.Generator().manual_seed(64)
    mk, ms = torch.randn(CK, READER_N, generator=g), 1 + torch.rand(READER_N, generator=g)
    qk, qe = torch.randn(CK, READER_Q, generator=g), torch.sigmoid(torch.randn(CK, READER_Q, generator=g))
    mv = torch.randn(2 * CV, READER_N, generator=g)
    return mk, ms, qk, qe, mv


def _shard_cfg(meta, world):
    cfg = dict(meta['configs']['50'], top_k=SHARD_TOP_K)
    return dict(cfg, num_prototypes=126) if world == 3 else cfg   # the prototypes must divide by the world


def _rank_main(rank, world, port, golden_dir, out_dir):
    for p in (ROOT, os.path.join(ROOT, 'tracking-anything-with-deva_b200')):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world, timeout=timedelta(seconds=60))
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    import deva.inference.sharded_core as sharded_core
    import deva.inference.sharded_memory as sharded_memory
    from deva.inference.sharded_core import ShardedDEVAInferenceCore
    from deva.inference.sharded_memory import ShardedBankReader, shard_bounds
    sharded_core.dist = sharded_memory.dist = StagedCollectives()
    res = {}
    mk, ms, qk, qe, mv = _reader_inputs()
    lo, hi = shard_bounds(READER_N, world, rank)
    reader = ShardedBankReader(CK, CV, 2, hi - lo, lo, dev, top_k=SHARD_TOP_K)
    reader.load(mk[:, lo:hi].to(dev), ms[lo:hi].to(dev), mv[:, lo:hi].to(dev))
    res['read'] = reader.read(qk.to(dev), qe.to(dev)).cpu()
    res['use'] = reader.use_cnt[:hi - lo].cpu()
    g, meta = _topk_clip(golden_dir)
    cfg = _shard_cfg(meta, world)
    np.random.seed(42)
    res['clip'] = _run_topk_clip(ShardedDEVAInferenceCore(_net(cfg, dev), cfg), g, dev)
    torch.save(res, os.path.join(out_dir, f'rank{rank}.pt'))
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()


@gpu
@pytest.mark.parametrize('world', [2, 3])
def test_sharded_ranks_at_top_k_64(world, golden_dir, tmp_path):
    """Every rank's ShardedBankReader read against float64, and the sharded core's session on every rank against the
    plain core at the same config."""
    import torch.multiprocessing as mp
    from deva.inference.inference_core import DEVAInferenceCore
    _nat()
    t0 = time.time()
    try:
        mp.spawn(_rank_main, args=(world, _free_port(), golden_dir, str(tmp_path)), nprocs=world, join=True)
    except Exception as e:
        if 'busy or unavailable' in str(e):
            pytest.skip('the device refuses a second context (exclusive-process compute mode)')
        raise
    ranks = [torch.load(os.path.join(str(tmp_path), f'rank{r}.pt')) for r in range(world)]
    print(f'[topk-wide] world {world}: {time.time() - t0:.1f} s for the spawn')
    mk, ms, qk, qe, mv = _reader_inputs()
    ref, use, _, _ = mm.read(mk.double(), ms.double(), qk.double(), qe.double(), mv.half().double(), SHARD_TOP_K)
    scale = max(1.0, float(ref.abs().max()))
    for r in range(world):
        err = float((ranks[r]['read'].double() - ref).abs().max()) / scale
        _report(f'world {world} rank {r} reader read-out vs float64 (relative)', err, READ_REL)
        assert err <= READ_REL
    use_all = torch.cat([ranks[r]['use'] for r in range(world)]).double()
    e_use = float((use_all - use).abs().max())
    _report(f'world {world} reader usage vs float64', e_use, 2e-4)
    assert e_use <= 2e-4
    g, meta = _topk_clip(golden_dir)
    cfg = _shard_cfg(meta, world)
    np.random.seed(42)
    plain = _run_topk_clip(DEVAInferenceCore(_net(cfg, 'cuda'), cfg), g, 'cuda')
    for r in range(1, world):
        for t, (a, b) in enumerate(zip(ranks[0]['clip']['probs'], ranks[r]['clip']['probs'])):
            assert torch.equal(a, b), f'rank {r} differs from rank 0 on frame {t}'
    per_frame = [float((a - b).abs().max()) for a, b in zip(ranks[0]['clip']['probs'], plain['probs'])]
    _report(f'world {world} clip max |prob - plain core| (worst frame {int(np.argmax(per_frame))})', max(per_frame),
            PROB_CLIP)
    assert max(per_frame) < PROB_CLIP
