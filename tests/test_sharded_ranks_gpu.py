"""The bank-sharded single-video mode (deva/inference/sharded_core.py, sharded_memory.py) on 2, 3 and 4 ranks that share
ONE GPU, every rank checked against float64 (memory level) and against the plain core (session level).

Nothing in the sharded mode needs a second device to be correct: it needs several ranks, each a process with its own
CUDA context, a process group, and peer memory mapped through CUDA IPC.  Only NCCL refuses two ranks on one device, so
each worker replaces the name ``dist`` as seen by the two product modules with ``StagedCollectives``: everything is
forwarded to ``torch.distributed`` (gloo) except ``all_gather_into_tensor``, ``all_reduce`` and ``all_to_all_single``,
which copy the CUDA tensor to the host, run the gloo collective there and copy the result back into the caller's tensor.
``PeerBuffers`` runs unmodified - ``peer_alloc``, ``all_gather_object`` of the IPC handles, ``peer_open`` of another
process's allocation, ``red.add`` from ``readout_sparse_scatter`` into the mapped pointers - so the IPC path is the real
one; only the transport of the small collectives differs from production.

Ordering.  The product relies on NCCL's stream order for two things: a rank's buffer is zeroed before any remote add
(the zeroing is enqueued before the candidate all-gather), and all adds are complete before the fence returns.  The
staged collectives synchronise the calling rank's stream in their ``.cpu()`` copy before the host collective starts, so
both hold here MORE strongly than in production: a missing stream dependency in the product would not show in this
file.  What does show is everything else: partitions, padding rows, slot ids, thresholds, prototype slices.

One spawn per world size runs every case of that world and saves each rank's raw outputs; the parent process draws the
same inputs from the same seeds, computes the references and asserts.  World 3 makes every partition ragged.  A worker
that raises ends the spawn (its siblings are terminated); a lock-step bug ends in the group's 60 s time-out, not a
hang.  Where the device refuses a second context (exclusive-process compute mode) the GPU tests skip with that reason.

Not covered here, by construction: NCCL transport, peer adds between DIFFERENT devices over NVLink, and any timing.
The sharded core supports ``incorporate_detection`` with purges (``purge_except`` + the re-partition in
``set_objects``); the detection session below drives it.
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
CK, CV, LP = 64, 128, 32
WORLDS = (2, 3, 4)
SIM_ABS = 1e-4            # similarity bound of tests/test_memory_kernels_gpu.py
W_ABS = 2e-5              # softmax weight bound of the memory-read tests
READ_REL = 1e-3           # read-out bound, relative to max(1, max |reference|)
USE_ABS = 2e-4            # usage (a sum of up to 1620 weights per slot)
SOFTMAX_REL = 2 * SIM_ABS + 2e-5   # consolidation: exp(+-2 SIM_ABS) and fp32 sums, as test_consolidation_dense_softmax
# The session bounds are measured figures (H100 80GB HBM3, 700 W) plus headroom.  One rank differs from the plain core by
# 2e-5.  Several ranks add their partial read-outs in fp32 in another order than one GEMM does: on the golden clip's first
# read 2 or 3 of 30 720 read-out elements land on the neighbouring fp16 value, everything else that enters the decoder is
# bit-identical, and the fp16 network turns that into 1.0e-4 .. 1.7e-4 of probability on that same frame.  It is the
# network's sensitivity to one fp16 ulp, not a property of the sharding, and it saturates at the stack's fp16 error.
PROB_CLIP = 2e-3          # |prob - plain core|, golden clip: measured 5.8e-4 .. 8.5e-4 at world 2, 3, 4 over two runs
PROB_REAL = 1e-3          # ... at 480 x 864 with evictions: measured 2.6e-4 .. 2.8e-4
PROB_DET = 1e-3           # ... in the detection session, up to the first propagated frame
SENSORY_REL = 1.5e-2      # sensory rows (fp16, in [-1, 1]) against the plain core's: measured 3.7e-3 .. 4.8e-3
PROB_REF = 2e-3           # |prob - reference fixture|: measured 6.7e-4 (world 4), 1.1e-3 (world 2); the plain core 9.4e-4


def _report(name, err, bound):
    print(f'[sharded-ranks] {name}: measured {err:.3e}, bound {bound:.3e}')


# ------------------------------------------------------------------------------------------------- staged collectives
class StagedCollectives:
    """``torch.distributed`` for a gloo group whose callers hold CUDA tensors: the three tensor collectives the sharded
    mode uses are staged through the host (gloo rejects a ``[world, ...]`` ``all_gather_into_tensor`` output, so that one
    runs as ``all_gather`` into the rows of the host copy); every other name is ``torch.distributed``'s own."""

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


def _init_group(rank, world, port):
    for p in (ROOT, os.path.join(ROOT, 'tracking-anything-with-deva_b200')):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world, timeout=timedelta(seconds=60))


def _staging_worker(rank, world, port, out_dir):
    _init_group(rank, world, port)
    st = StagedCollectives()
    res = {}
    for name, dtype in (('f32', torch.float32), ('f16', torch.float16), ('i32', torch.int32)):
        mine = (torch.arange(10).view(2, 5) + 100 * rank).to(dtype)
        out = torch.full((world, 2, 5), -1, dtype=dtype)
        st.all_gather_into_tensor(out, mine)
        s, m = mine.clone(), mine.clone()
        st.all_reduce(s)
        st.all_reduce(m, op=dist.ReduceOp.MAX)
        send = (torch.arange(world * 3).view(world, 3) + 100 * rank).to(dtype)
        recv = torch.full_like(send, -1)
        st.all_to_all_single(recv, send)
        res[name] = dict(gather=out, sum=s, max=m, a2a=recv)
    res['world'] = st.get_world_size()  # a forwarded name
    torch.save(res, os.path.join(out_dir, f'rank{rank}.pt'))
    dist.barrier()
    dist.destroy_process_group()


def test_staged_collectives_on_three_cpu_ranks(tmp_path):
    """The helper itself, on CPU tensors: each staged collective equals the obvious torch expression."""
    import torch.multiprocessing as mp
    world = 3
    mp.spawn(_staging_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    for rank in range(world):
        res = torch.load(os.path.join(tmp_path, f'rank{rank}.pt'))
        assert res['world'] == world
        for name, dtype in (('f32', torch.float32), ('f16', torch.float16), ('i32', torch.int32)):
            mine = [(torch.arange(10).view(2, 5) + 100 * r).to(dtype) for r in range(world)]
            got = res[name]
            assert got['gather'].dtype == dtype
            assert torch.equal(got['gather'], torch.stack(mine)), (rank, name)        # row r = rank r's tensor
            assert torch.equal(got['sum'], torch.stack(mine).sum(0).to(dtype)), (rank, name)
            assert torch.equal(got['max'], mine[-1]), (rank, name)
            want = torch.stack([(torch.arange(world * 3).view(world, 3) + 100 * r).to(dtype)[rank] for r in range(world)])
            assert torch.equal(got['a2a'], want), (rank, name)                         # row r = what rank r sent to me


# ------------------------------------------------------------------------------------------------- inputs (one seed)
READ_CASES = [
    # n slots, k objects, top_k, query counts of successive reads on the same reader
    dict(name='ragged', n=203, k=5, top_k=30, qs=(37, 50)),   # n not a multiple of 8 * world; a new Q reopens the peers
    dict(name='tiny', n=10, k=1, top_k=6, qs=(20, )),         # k_loc < top_k, trailing ranks without slots or objects
    dict(name='short', n=44, k=4, top_k=30, qs=(33, )),       # every shard shorter than top_k; world 4: last shard empty
    dict(name='groups', n=120, k=258, top_k=30, qs=(40, )),   # more objects than one read-out launch takes
    dict(name='frame', n=5003, k=3, top_k=30, qs=(1620, )),   # shards longer than top_k, a 480 x 864 frame of queries
]


def _read_inputs(i):
    c = READ_CASES[i]
    g = torch.Generator().manual_seed(100 + i)
    mk, ms = torch.randn(CK, c['n'], generator=g), 1 + torch.rand(c['n'], generator=g)
    mv = torch.randn(c['k'] * CV, c['n'], generator=g)
    queries = [(torch.randn(CK, q, generator=g), torch.sigmoid(torch.randn(CK, q, generator=g))) for q in c['qs']]
    return mk, ms, mv, queries


CONS_P = 24          # global prototypes: 12, 8 and 6 per rank
CONS_PRE, CONS_POST = 5, 3   # bank tokens in front of / behind the candidates: the window has 5 lead slots
CONS_CASES = [dict(name='spread', n=1003), dict(name='starved', n=1003), dict(name='ties', n=602)]
CONS_TIED = 10       # 'ties': 20 candidates above, 10 exactly at 0.5, the rest below; 4 of the 10 are chosen


def _cons_inputs(i, world):
    """Candidates of all ranks: keys close enough that every prototype's softmax spreads over all ranks' candidates."""
    c = CONS_CASES[i]
    n = c['n']
    g = torch.Generator().manual_seed(200 + i)
    key, shr = 0.3 * torch.randn(CK, n, generator=g), 1 + torch.rand(n, generator=g)
    sel = torch.sigmoid(torch.randn(CK, n, generator=g))
    val = torch.randn(3 * CV, n, generator=g)
    life = 1 + torch.randint(0, 5, (n, ), generator=g).float()
    u = (torch.randperm(n, generator=g) + 1).float() / n         # distinct, 1 / n apart
    if c['name'] == 'starved':                                   # the last rank owns none of the chosen prototypes
        from deva.inference.sharded_core import token_bounds
        lo, hi = token_bounds(n, world, world - 1)
        u[lo:hi] *= 0.01
    use = u * life
    if c['name'] == 'ties':
        order = torch.randperm(n, generator=g)
        top, tied = order[:CONS_P - 4], order[CONS_P - 4:CONS_P - 4 + CONS_TIED]
        use = 0.4 * u * life
        use[top] = (0.6 + 0.01 * torch.arange(CONS_P - 4)) * life[top]
        use[tied], life[tied] = 2.0, 4.0
    return key, shr, sel, val, use, life


EVICT_KEEP = 30      # local max_size: the ranks together keep at most 30 * world
EVICT_CASES = ['skewed', 'ties']


def _evict_sizes(world):
    return [40 + 5 * r for r in range(world)]   # different local sizes: the gathered usage is padded to the longest


def _evict_inputs(i, world):
    sizes = _evict_sizes(world)
    n = sum(sizes)
    g = torch.Generator().manual_seed(300 + i)
    key, val = torch.randn(n, CK, generator=g), torch.randn(2 * CV, n, generator=g)
    use = (torch.randperm(n, generator=g) + 1).float()   # life = 4: usage = use / 4 exactly, in fp32 and fp64
    use[:sizes[0]] += n                                  # rank 0 keeps everything, the other ranks pay for it
    drop = n - EVICT_KEEP * world
    if EVICT_CASES[i] == 'ties':                         # five slots AT the global threshold: strict '>' drops them all
        order = torch.argsort(use)
        use[order[drop - 3:drop + 2]] = float(use[order[drop - 1]])
    return key, val, use


CLIP_CFG = {3: dict(num_prototypes=126)}   # must divide by the world; 2 and 4 run the fixture's own config


def _clip(golden_dir):
    g = {k: torch.from_numpy(v) for k, v in np.load(os.path.join(golden_dir, 'vos_steps.npz')).items()}
    meta = json.load(open(os.path.join(golden_dir, 'vos_steps.json')))
    return g, meta


REAL_CFG = dict(mem_every=1, max_mid_term_frames=4, min_mid_term_frames=2, num_prototypes=128,
                max_long_term_elements=240)   # 8 frames: consolidation after frames 3, 5, 7; eviction at 5 and 7
REAL_FRAMES, REAL_H, REAL_W = 8, 480, 864


def _real_inputs():
    g = torch.Generator().manual_seed(400)
    up = lambda t: torch.nn.functional.interpolate(t, size=(REAL_H, REAL_W), mode='bilinear', align_corners=False)
    base = up(torch.randn(1, 3, 30, 54, generator=g))[0]
    frames = [base + 0.15 * t * up(torch.randn(1, 3, 15, 27, generator=g))[0] for t in range(REAL_FRAMES)]
    mask = torch.zeros(REAL_H, REAL_W, dtype=torch.long)
    for o, (y, x) in enumerate([(20, 30), (40, 500), (250, 100), (260, 420), (300, 700)]):
        mask[y:y + 150, x:x + 140] = o + 1
    return frames, mask


def _det_inputs():
    g = torch.Generator().manual_seed(8)
    h, w = 96, 128
    img = torch.randn(3, h, w, generator=g)
    img2 = img + 0.05 * torch.randn(3, h, w, generator=g)
    det = torch.zeros(h, w, dtype=torch.long)
    det[8:40, 8:60] = 5
    det[50:90, 60:120] = 6
    det2 = torch.zeros(h, w, dtype=torch.long)
    det2[8:40, 8:60] = 77
    return img, img2, det, det2


# ------------------------------------------------------------------------------------------------- sessions (any core)
def _net(cfg, dev):
    from deva.model.network import DEVA
    from deva.model.param_spec import synthetic_state_dict
    net = DEVA(cfg).to(dev).eval()
    net.load_weights({k: v.to(dev) for k, v in synthetic_state_dict(seed=1).items()})
    return net


def _sizes(core):
    mem = core.memory
    return {str(b): [mem.work_mem.size(b), mem.long_mem.size(b)] for b in mem.work_mem.buckets}


def _sensory(core):
    mem = core.memory
    block = None if mem._sensory_block is None else mem._sensory_block.float().cpu()
    return dict(ids=list(mem._sensory_ids), own=list(mem.own_ids()) if hasattr(mem, 'own_ids') else None, block=block)


def _run_clip(core, g, dev):
    T = g['frames'].shape[0]
    out = dict(probs=[], sizes=[], sensory={}, reads=[])
    read = core.memory.match_memory

    def recording_read(key, selection):   # [K (own), CV, h, w] per read, in temporary-id order
        got = read(key, selection)
        out['reads'].append((torch.stack(list(got.values())) if isinstance(got, dict) else got[0]).float().cpu())
        return got
    core.memory.match_memory = recording_read
    for t in range(T):
        img = g['frames'][t].to(dev)
        if t == 0:
            p = core.step(img, g['mask0'].to(dev), [1, 2])
        elif t == 6:
            p = core.step(img, g['mask6'].to(dev), [7])
        else:
            p = core.step(img, end=(t == T - 1))
        out['probs'].append(p.float().cpu())
        out['sizes'].append(_sizes(core))
        if t in (0, 5, 6, 10):
            out['sensory'][t] = _sensory(core)
    return out


def _run_real(core, dev):
    frames, mask = _real_inputs()
    out = dict(probs=[], sizes=[])
    for t, img in enumerate(frames):
        p = core.step(img.to(dev), mask.to(dev), [1, 2, 3, 4, 5]) if t == 0 else core.step(img.to(dev))
        out['probs'].append(p.float().cpu())
        out['sizes'].append(_sizes(core))
    return out


def _run_detections(core, dev):
    """Two objects enter by detection, a third replaces them, the first two are purged after missing two detections."""
    from deva.inference.object_info import ObjectInfo
    img, img2, det, det2 = (t.to(dev) for t in _det_inputs())
    out = dict(probs=[], ids=[], sensory=[])

    def keep(p):
        out['probs'].append(p.float().cpu())
        out['ids'].append(list(core.object_manager.all_obj_ids))
        out['sensory'].append(_sensory(core))
    keep(core.incorporate_detection(img, det, [ObjectInfo(5), ObjectInfo(6)]))
    keep(core.step(img2))
    for _ in range(3):
        keep(core.incorporate_detection(img, det2, [ObjectInfo(77)]))
    keep(core.step(img2))
    return out


def _det_cfg(meta):
    return dict(meta['config'], mem_every=5, max_long_term_elements=9600, num_prototypes=120,
                max_missed_detection_count=1, max_num_objects=-1)


# ------------------------------------------------------------------------------------------------- the ranks
def _rank_reads(rank, world, dev):
    from deva.inference.sharded_memory import ShardedBankReader, shard_bounds
    res = []
    for i, c in enumerate(READ_CASES):
        mk, ms, mv, queries = _read_inputs(i)
        lo, hi = shard_bounds(c['n'], world, rank)
        rd = ShardedBankReader(CK, CV, c['k'], hi - lo, lo, dev, top_k=c['top_k'])
        rd.load(mk[:, lo:hi].to(dev), ms[lo:hi].to(dev), mv[:, lo:hi].to(dev))
        reads = []
        for qk, qe in queries:
            q = qk.shape[1]
            one = {}
            for kind, fn in (('read', rd.read), ('scatter', rd.read_scatter)):
                rd.use_cnt.zero_()
                out = fn(qk.to(dev), qe.to(dev)).clone()
                one[kind] = dict(out=out.cpu(), use=rd.use_cnt[:hi - lo].cpu(),
                                 sel=rd._buf('g_sel', (q, LP), torch.int32).cpu(),
                                 w=rd._buf('g_w', (q, LP), torch.float32).cpu(), own=rd.objects_of(rank))
            reads.append(one)
        res.append(reads)
        torch.cuda.synchronize()
        dist.barrier()  # nobody releases its buffer while a peer still has it mapped for this reader
    return res


def _memory_manager(world):
    from deva.inference.sharded_core import ShardedMemoryManager
    cfg = dict(key_dim=CK, value_dim=CV, top_k=30, enable_long_term=True, enable_long_term_count_usage=True,
               chunk_size=-1, max_mid_term_frames=4, min_mid_term_frames=2, num_prototypes=CONS_P,
               max_long_term_elements=240)
    mem = ShardedMemoryManager(cfg)
    assert mem.world == world and mem.num_prototypes == CONS_P // world
    mem.CK, mem.CV = CK, CV
    return mem


def _rank_consolidation(rank, world, dev):
    from deva.inference.memory_bank import BucketBank
    from deva.inference.sharded_core import token_bounds
    mem = _memory_manager(world)
    res = []
    for i, c in enumerate(CONS_CASES):
        key, shr, sel, val, use, life = _cons_inputs(i, world)
        lo, hi = token_bounds(c['n'], world, rank)
        n_loc = hi - lo
        m = CONS_PRE + n_loc + CONS_POST
        g = torch.Generator().manual_seed(900 + rank)   # the tokens around the candidates differ per rank
        pad = lambda t, fill: torch.cat([fill(t[..., :CONS_PRE]), t[..., lo:hi], fill(t[..., :CONS_POST])], -1).to(dev)
        rnd = lambda t: torch.randn(t.shape, generator=g)
        bank = BucketBank([1, 2, 3], CK, CV, 64, m + 8, dev)
        bank.append_work(pad(key, rnd), pad(shr, lambda t: 1 + torch.rand(t.shape, generator=g)),
                         pad(sel, lambda t: torch.sigmoid(rnd(t))),
                         {o: pad(val[j * CV:(j + 1) * CV], rnd).contiguous() for j, o in enumerate([1, 2, 3])})
        bank.keep_objects({1, 3})   # a purged object in the middle: value rows 0 and 2 are the live ones
        c0 = bank.base + CONS_PRE
        c1 = c0 + n_loc
        bank.use_cnt[bank.base:bank.hi] = 1e6   # the neighbours would win every prototype if the window were off by one
        bank.life_cnt[bank.base:bank.hi] = 1.0
        bank.use_cnt[c0:c1], bank.life_cnt[c0:c1] = use[lo:hi].to(dev), life[lo:hi].to(dev)
        pk, pv, ps = mem.consolidation(bank, c0, c1)
        res.append(dict(key=pk.cpu(), val=pv.cpu(), shr=ps.cpu()))
    return res


def _rank_eviction(rank, world, dev):
    from deva.inference.memory_bank import BucketBank
    mem = _memory_manager(world)
    sizes = _evict_sizes(world)
    lo = sum(sizes[:rank])
    hi = lo + sizes[rank]
    res = []
    for i in range(len(EVICT_CASES)):
        key, val, use = _evict_inputs(i, world)
        bank = BucketBank([1, 2], CK, CV, 64, 64, dev)
        ids = torch.arange(lo, hi).float() + 1   # the shrinkage column carries each slot's global id
        bank.prepend_long(key[lo:hi].to(dev).contiguous(), ids.to(dev), val[:, lo:hi].to(dev).contiguous())
        assert bank.long_size == hi - lo
        bank.use_cnt[bank.lo:bank.base] = use[lo:hi].to(dev)
        bank.life_cnt[bank.lo:bank.base] = 4.0
        before = mem._long_size(bank)
        mem._evict_long(bank, EVICT_KEEP)
        res.append(dict(ids=bank.raw_shr[bank.lo:bank.base].cpu(), key=bank.raw_key[bank.lo:bank.base].cpu(),
                        val=bank.values[:, :, bank.lo:bank.base].float().cpu(), use=bank.use_cnt[bank.lo:bank.base].cpu(),
                        before=before, after=mem._long_size(bank), local=bank.long_size))
    return res


REPART_IDS = [[10, 11], [10, 11, 12, 13, 14], [11, 13, 14], [14], [14, 20, 21, 22, 23, 24, 25], [14, 20, 21, 22, 23, 24, 25], []]
REPART_HW = (3, 5)


def _repart_row(obj):
    """Object ``obj``'s sensory row: exact in fp16, different at every position."""
    h, w = REPART_HW
    return ((obj * 8 + torch.arange(CV * h * w) % 7).float() / 512).view(CV, h, w)


def _rank_repartition(rank, world, dev):
    """``set_objects`` through growth, a purge in the middle, one object, more objects than ranks, no change, none: after
    each call every own row is overwritten with that object's pattern, as a decoded frame would."""
    mem = _memory_manager(world)
    key = torch.zeros(1, CK, *REPART_HW, device=dev)
    res = []
    for ids in REPART_IDS:
        mem.set_objects(ids, key)
        block = mem._sensory_block
        res.append(dict(ids=list(mem._sensory_ids), own=list(mem.own_ids()),
                        block=None if block is None else block.float().cpu()))
        for i, o in enumerate(mem._sensory_ids):
            block[i] = _repart_row(o).to(dev)
    return res


def _rank_main(rank, world, port, golden_dir, out_dir):
    _init_group(rank, world, port)
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    import deva.inference.sharded_core as sharded_core
    import deva.inference.sharded_memory as sharded_memory
    from deva.inference.sharded_core import ShardedDEVAInferenceCore
    sharded_core.dist = sharded_memory.dist = StagedCollectives()
    res, clock = {}, {}

    def timed(name, fn):
        t0 = time.time()
        res[name] = fn()
        torch.cuda.synchronize()
        clock[name] = time.time() - t0

    timed('reads', lambda: _rank_reads(rank, world, dev))
    timed('consolidation', lambda: _rank_consolidation(rank, world, dev))
    timed('eviction', lambda: _rank_eviction(rank, world, dev))
    timed('repartition', lambda: _rank_repartition(rank, world, dev))
    g, meta = _clip(golden_dir)
    cfg = dict(meta['config'], **CLIP_CFG.get(world, {}))
    np.random.seed(42)
    timed('clip', lambda: _run_clip(ShardedDEVAInferenceCore(_net(cfg, dev), cfg), g, dev))
    cfg = _det_cfg(meta)
    np.random.seed(42)   # fresh ids of unmatched detections are random draws
    timed('detections', lambda: _run_detections(ShardedDEVAInferenceCore(_net(cfg, dev), cfg), dev))
    if world in (2, 4):
        cfg = dict(meta['config'], **REAL_CFG)
        timed('real', lambda: _run_real(ShardedDEVAInferenceCore(_net(cfg, dev), cfg), dev))
    res['clock'] = clock
    torch.save(res, os.path.join(out_dir, f'rank{rank}.pt'))
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()


_RUNS = {}


def _ranks(world, golden_dir, tmp_path_factory):
    """Every rank's saved outputs for ``world``; the processes are spawned once per world size and all have exited."""
    if world not in _RUNS:
        import torch.multiprocessing as mp
        out_dir = str(tmp_path_factory.mktemp(f'world{world}'))
        t0 = time.time()
        try:
            mp.spawn(_rank_main, args=(world, _free_port(), golden_dir, out_dir), nprocs=world, join=True)
            _RUNS[world] = [torch.load(os.path.join(out_dir, f'rank{r}.pt')) for r in range(world)]
            clock = _RUNS[world][0]['clock']
            print(f'[sharded-ranks] world {world}: {time.time() - t0:.1f} s for the spawn; rank 0: ' +
                  ', '.join(f'{k} {v:.1f} s' for k, v in clock.items()))
        except Exception as e:  # kept: the other tests of this world report it without spawning again
            _RUNS[world] = e
    got = _RUNS[world]
    if isinstance(got, Exception):
        if 'busy or unavailable' in str(got):
            pytest.skip('the device refuses a second context (exclusive-process compute mode)')
        raise got
    return got


_PLAIN = {}


def _plain(name, cfg, run):
    """The plain single-GPU core with the same config, in this process."""
    key = (name, json.dumps(cfg, sort_keys=True))
    if key not in _PLAIN:
        from deva.inference.inference_core import DEVAInferenceCore
        np.random.seed(42)
        _PLAIN[key] = run(DEVAInferenceCore(_net(cfg, 'cuda'), cfg))
    return _PLAIN[key]


def _check_probs(name, ranks, plain, bound, upto=None):
    """Every rank bit-identical (they all run ``probabilities`` on the same gathered logits); max |prob - plain core| over
    the first ``upto`` frames (default: all)."""
    for r, got in enumerate(ranks[1:], 1):
        for t, (a, b) in enumerate(zip(ranks[0]['probs'], got['probs'])):
            assert torch.equal(a, b), f'{name}: rank {r} differs from rank 0 on frame {t}'
    assert len(ranks[0]['probs']) == len(plain['probs'])
    assert all(a.shape == b.shape for a, b in zip(ranks[0]['probs'], plain['probs']))
    per_frame = [float((a - b).abs().max()) for a, b in zip(ranks[0]['probs'], plain['probs'])][:upto]
    _report(f'{name} max |prob - plain core| (worst frame {int(np.argmax(per_frame))})', max(per_frame), bound)
    assert max(per_frame) < bound, per_frame


def _check_sensory(steps, world):
    """steps: [(plain core's snapshot, every rank's snapshot)] in time order.  Each rank holds exactly the objects it owns,
    and its rows are the plain core's rows of those objects.  -> (worst relative difference, rows that changed rank between
    consecutive snapshots, rank-steps that own nothing)."""
    from deva.inference.sharded_core import object_bounds
    worst, moved, idle, where = 0.0, 0, 0, {}
    for ps, rs in steps:
        ids = ps['ids']
        for r in range(world):
            s = rs[r]
            lo, hi = object_bounds(len(ids), world, r)
            assert s['ids'] == s['own'] == ids[lo:hi], f'rank {r} holds {s["ids"]}, owns {ids[lo:hi]}'
            moved += sum(1 for o in s['ids'] if where.get(o, r) != r)
            where.update({o: r for o in s['ids']})
            if hi == lo:
                idle += 1
                assert s['block'] is None
                continue
            want = ps['block'][lo:hi]
            assert s['block'].shape == want.shape
            worst = max(worst, float((s['block'] - want).abs().max()) / max(1.0, float(want.abs().max())))
    return worst, moved, idle


# ------------------------------------------------------------------------------------------------- memory level
@gpu
@pytest.mark.parametrize('world', WORLDS)
def test_reads_match_float64(world, golden_dir, tmp_path_factory):
    """``ShardedBankReader.read`` / ``.read_scatter``: the global top-k set, its weights, the read-out and each rank's usage
    against the unsharded float64 read."""
    from deva.inference.sharded_memory import shard_bounds
    ranks = _ranks(world, golden_dir, tmp_path_factory)
    for i, c in enumerate(READ_CASES):
        mk, ms, mv, queries = _read_inputs(i)
        n, k, top_k = c['n'], c['k'], c['top_k']
        bounds = [shard_bounds(n, world, r) for r in range(world)]
        per = -(-k // world)
        for j, (qk, qe) in enumerate(queries):
            q = qk.shape[1]
            name = f"world {world} '{c['name']}' n={n} K={k} Q={q}"
            sim = mm.similarity(mk.double().cuda(), ms.double().cuda(), qk.double().cuda(), qe.double().cuda())  # [n, q]
            vals, ref_idx = torch.topk(sim, k=top_k, dim=0)
            for kind in ('read', 'scatter'):
                got = [ranks[r]['reads'][i][j][kind] for r in range(world)]
                for r in range(1, world):  # the same merge of the same gathered lists
                    assert torch.equal(got[r]['sel'], got[0]['sel']) and torch.equal(got[r]['w'], got[0]['w'])
                sel = got[0]['sel'][:, :top_k].long().cuda()
                assert int(sel.min()) >= 0 and int(sel.max()) < n, f'{name}: a slot id outside the bank'
                srt = torch.sort(sel, 1)[0]
                assert bool((srt[:, 1:] != srt[:, :-1]).all()), f'{name}: a slot was selected twice'
                same = (torch.sort(ref_idx.t(), 1)[0] == srt).all(1)
                gap = vals[top_k - 1] - (sim.sort(0, descending=True)[0][top_k] if n > top_k else -float('inf'))
                assert bool((same | (gap < 2e-4)).all()), f'{name}: top-k sets differ on {int((~same).sum())} queries'
                # the float64 read over the selected slots (= the float64 read wherever the sets are equal)
                w64 = torch.softmax(sim.t().gather(1, sel), 1)
                err_w = float((got[0]['w'][:, :top_k].double().cuda() - w64).abs().max())
                aff = torch.zeros(q, n, dtype=torch.float64, device='cuda').scatter_(1, sel, w64)
                ref = mv.double().cuda() @ aff.t()
                scale = max(1.0, float(ref.abs().max()))
                if kind == 'read':
                    for r in range(1, world):
                        assert torch.equal(got[r]['out'], got[0]['out']), f'{name}: rank {r} read differs from rank 0'
                    assert tuple(got[0]['out'].shape) == (k * CV, q)
                    err = float((got[0]['out'].double().cuda() - ref).abs().max()) / scale
                else:
                    err = 0.0
                    for r in range(world):
                        lo, hi = min(k, r * per), min(k, (r + 1) * per)
                        assert got[r]['own'] == (lo, hi)
                        assert tuple(got[r]['out'].shape) == ((hi - lo) * CV, q), f'{name}: rank {r} holds other objects'
                        if hi > lo:
                            e = float((got[r]['out'].double().cuda() - ref[lo * CV:hi * CV]).abs().max())
                            err = max(err, e / scale)
                use = torch.cat([got[r]['use'] for r in range(world)])
                assert [int(g['use'].numel()) for g in got] == [hi - lo for lo, hi in bounds]
                err_u = float((use.double().cuda() - aff.sum(0)).abs().max())
                _report(f'{name} {kind}: weights', err_w, W_ABS)
                _report(f'{name} {kind}: read-out / max(1, |ref|)', err, READ_REL)
                _report(f'{name} {kind}: usage of own slots', err_u, USE_ABS)
                assert err_w < W_ABS and err < READ_REL and err_u < USE_ABS, name


@gpu
@pytest.mark.parametrize('world', WORLDS)
def test_consolidation_matches_float64(world, golden_dir, tmp_path_factory):
    """``ShardedMemoryManager.consolidation``: the ranks' slices together are the float64 prototypes of the float64 top-P
    usage over all ranks' candidates, rank r holding ``[r * p_loc, (r + 1) * p_loc)``."""
    from deva.inference.sharded_core import token_bounds
    ranks = _ranks(world, golden_dir, tmp_path_factory)
    p_loc = CONS_P // world
    for i, c in enumerate(CONS_CASES):
        name = f"world {world} consolidation '{c['name']}' n={c['n']}"
        key, shr, sel, val, use, life = (t.cuda() for t in _cons_inputs(i, world))
        got = [ranks[r]['consolidation'][i] for r in range(world)]
        assert all(tuple(g['key'].shape) == (p_loc, CK) and tuple(g['val'].shape) == (2 * CV, p_loc) and
                   tuple(g['shr'].shape) == (p_loc, ) for g in got)
        pk = torch.cat([g['key'] for g in got]).cuda()      # rank-major = the global prototype order
        pv = torch.cat([g['val'] for g in got], 1).cuda()
        ps = torch.cat([g['shr'] for g in got]).cuda()
        hit = (key.t().unsqueeze(0) == pk.unsqueeze(1)).all(-1)   # keys are gathered rows: exact
        assert bool((hit.sum(1) == 1).all()), f'{name}: a prototype key is not a candidate row'
        chosen = hit.long().argmax(1)
        u64 = use.double() / life.double()
        if c['name'] == 'ties':
            assert len(set(chosen.tolist())) == CONS_P
            above = set(torch.nonzero(u64 > 0.5).view(-1).tolist())
            tied = set(torch.nonzero(u64 == 0.5).view(-1).tolist())
            assert len(above) == CONS_P - 4 and len(tied) == CONS_TIED
            assert chosen[:CONS_P - 4].tolist() == torch.topk(u64, CONS_P - 4)[1].tolist()
            assert set(chosen[CONS_P - 4:].tolist()) <= tied, f'{name}: a candidate below the tie was chosen'
        else:
            assert chosen.tolist() == torch.topk(u64, CONS_P)[1].tolist(), f'{name}: not the float64 top-P in order'
        owners = [sum(1 for t in chosen.tolist() if token_bounds(c['n'], world, r)[0] <= t <
                      token_bounds(c['n'], world, r)[1]) for r in range(world)]
        if c['name'] == 'starved':
            assert owners[-1] == 0
        sim = mm.similarity(key.double(), shr.double(), pk.t().double(), sel.t()[chosen].t().double())   # [n, P]
        p64 = torch.softmax(sim, 0)
        spread = float(p64.max(0)[0].max())
        shr64 = p64.t() @ shr.double()
        live = torch.cat([val[:CV], val[2 * CV:]]).double()
        val64, mag = live @ p64, live.abs() @ p64
        err_s = float(((ps.double() - shr64).abs() / shr64).max())
        # values and probabilities are stored in fp16 (2^-11 relative each) on top of the softmax's own error
        worst = float(((pv.double() - val64).abs() / (mag * (2.0 ** -10 + SOFTMAX_REL) + 1e-6)).max())
        _report(f'{name} (owners {owners}, largest probability {spread:.2f}): shrinkage, relative', err_s, SOFTMAX_REL)
        _report(f'{name}: values (err / bound)', worst, 1.0)
        assert err_s < SOFTMAX_REL and worst <= 1.0, name


@gpu
@pytest.mark.parametrize('world', WORLDS)
def test_eviction_keeps_what_the_unsharded_bank_keeps(world, golden_dir, tmp_path_factory):
    """``_evict_long`` against ``BucketBank.evict_long``'s rule on the concatenated bank: keep usage > the
    (n - max_size)-th smallest, strictly (quirk Q5), with and without ties at the threshold; ``_long_size``."""
    ranks = _ranks(world, golden_dir, tmp_path_factory)
    sizes = _evict_sizes(world)
    for i, case in enumerate(EVICT_CASES):
        name = f"world {world} eviction '{case}'"
        key, val, use = _evict_inputs(i, world)
        n = sum(sizes)
        usage = use.double() / 4
        thr = torch.sort(usage)[0][n - EVICT_KEEP * world - 1]
        keep = usage > thr
        kept_total = 0
        for r in range(world):
            got = ranks[r]['eviction'][i]
            lo = sum(sizes[:r])
            want = torch.nonzero(keep[lo:lo + sizes[r]]).view(-1) + lo
            assert (got['ids'] - 1).long().tolist() == want.tolist(), f'{name}: rank {r} kept other slots'
            assert got['local'] == int(want.numel())
            assert torch.equal(got['key'], key[want]) and torch.equal(got['use'], use[want])
            assert torch.equal(got['val'].reshape(2 * CV, -1), val[:, want].half().float())
            kept_total += got['local']
            assert got['before'] == n // world
        assert kept_total == int(keep.sum()) <= EVICT_KEEP * world
        assert kept_total == EVICT_KEEP * world - (2 if case == 'ties' else 0)
        assert all(ranks[r]['eviction'][i]['after'] == kept_total // world for r in range(world))
        per_rank = [ranks[r]['eviction'][i]['local'] for r in range(world)]
        assert per_rank[0] == sizes[0] and len(set(per_rank)) > 1   # a global threshold, not one per rank
        _report(f'{name}: kept per rank {per_rank} of {sizes}, all exact', 0.0, 0.0)


@gpu
@pytest.mark.parametrize('world', WORLDS)
def test_repartition_moves_sensory_rows_exactly(world, golden_dir, tmp_path_factory):
    """``set_objects``: each rank ends with the rows of ``own_ids()``; a known object's row arrives bit for bit (fp16
    transport of fp16-exact patterns) from whichever rank held it, a new object's row is zero."""
    from deva.inference.sharded_core import object_bounds
    ranks = [r['repartition'] for r in _ranks(world, golden_dir, tmp_path_factory)]
    known, where, moved, idle = set(), {}, 0, 0
    for t, ids in enumerate(REPART_IDS):
        for r in range(world):
            s = ranks[r][t]
            lo, hi = object_bounds(len(ids), world, r)
            assert s['ids'] == s['own'] == ids[lo:hi], f'step {t} rank {r} holds {s["ids"]}, owns {ids[lo:hi]}'
            if hi == lo:
                idle += 1
                assert s['block'] is None
                continue
            assert tuple(s['block'].shape) == (hi - lo, CV, *REPART_HW)
            for i, o in enumerate(s['ids']):
                want = _repart_row(o) if o in known else torch.zeros(CV, *REPART_HW)
                assert torch.equal(s['block'][i], want), f'step {t} rank {r}: the row of object {o} is not its own'
                moved += int(where.get(o, r) != r)
                where[o] = r
        known = set(ids)
    assert moved >= 2 and idle >= world
    _report(f'world {world} re-partition: {moved} rows changed rank, {idle} rank-steps without objects, all exact', 0.0, 0.0)


# ------------------------------------------------------------------------------------------------- session level
@gpu
@pytest.mark.parametrize('world', WORLDS)
def test_golden_clip_matches_plain_core(world, golden_dir, tmp_path_factory):
    """The 16-frame clip (objects 1, 2 at frame 0, 7 at frame 6, one consolidation) on every rank against the plain core
    with the same config: probabilities, per-rank bank sizes, and the sensory rows the frame-6 re-partition moved."""
    from deva.inference.sharded_core import object_bounds, token_bounds
    ranks = [r['clip'] for r in _ranks(world, golden_dir, tmp_path_factory)]
    g, meta = _clip(golden_dir)
    cfg = dict(meta['config'], **CLIP_CFG.get(world, {}))
    plain = _plain('clip', cfg, lambda core: _run_clip(core, g, 'cuda'))
    _check_probs(f'world {world} golden clip', ranks, plain, PROB_CLIP)
    if cfg == meta['config']:
        assert plain['sizes'] == meta['sizes']
        ref = max(float((a - g[f'prob_{t:02d}']).abs().max()) for t, a in enumerate(ranks[0]['probs']))
        _report(f'world {world} golden clip max |prob - reference fixture|', ref, PROB_REF)
        assert ref < PROB_REF
    # the first read (frame 1) sees the same bank in both cores - frame 0's values come from the given mask - so each rank's
    # read-out must be the plain core's rows of its objects up to the fp32 order of the partial sums, i.e. one fp16 ulp
    assert len(plain['reads']) == len(ranks[0]['reads']) == len(plain['probs']) - 1
    want = plain['reads'][0]
    worst, flipped, total = 0.0, 0, 0
    for r in range(world):
        lo, hi = object_bounds(want.shape[0], world, r)
        got = ranks[r]['reads'][0]
        assert got.shape == want[lo:hi].shape, f'rank {r} read {tuple(got.shape)}, owns objects [{lo}, {hi})'
        if hi > lo:
            err = (got - want[lo:hi]).abs()
            worst = max(worst, float((err / (want[lo:hi].abs() * 2.0 ** -10 + 2.0 ** -24)).max()))
            flipped, total = flipped + int((err > 0).sum()), total + err.numel()
    _report(f'world {world} golden clip frame 1 read-out vs plain core, in fp16 ulps ({flipped} of {total} elements differ)',
            worst, 1.0)
    assert worst <= 1.0
    hw = plain['sizes'][0]['0'][0]
    for r in range(world):
        t0, t1 = token_bounds(hw, world, r)
        want = [{b: [w // hw * (t1 - t0), l // world] for b, (w, l) in s.items()} for s in plain['sizes']]
        assert ranks[r]['sizes'] == want, f'rank {r}: bank sizes are not its token slice of the plain bank'
    assert any(l for s in plain['sizes'] for _, l in s.values()), 'the clip consolidates'
    # objects [1, 2] before frame 6 and [1, 2, 7] after, in blocks of ceil(K / world): at world 2 object 2 changes rank, at
    # world 3 and 4 a rank that owned nothing (k_own == 0) starts to own object 7
    steps = [(plain['sensory'][t], [ranks[r]['sensory'][t] for r in range(world)]) for t in (0, 5, 6, 10)]
    assert _check_sensory(steps[:1], world)[0] == 0.0, 'frame 0 (the given mask, no read) is not bit-identical'
    worst, moved, idle = _check_sensory(steps, world)
    assert moved >= (1 if world == 2 else 0) and idle >= (1 if world > 2 else 0)
    _report(f'world {world} golden clip sensory rows vs plain core, relative ({moved} rows changed rank, {idle} rank-steps '
            f'without objects)', worst, SENSORY_REL)
    assert worst < SENSORY_REL


@gpu
@pytest.mark.parametrize('world', WORLDS)
def test_detection_session_with_purge_matches_plain_core(world, golden_dir, tmp_path_factory):
    """``incorporate_detection``: objects 5 and 6 enter, 77 joins, 5 and 6 are purged - the object list shrinks from three
    to one, so the sensory rows are re-partitioned and most ranks end up owning nothing."""
    ranks = [r['detections'] for r in _ranks(world, golden_dir, tmp_path_factory)]
    _, meta = _clip(golden_dir)
    plain = _plain('detections', _det_cfg(meta), lambda core: _run_detections(core, 'cuda'))
    ids = plain['ids']
    assert ids[0] == [6, 5] and max(len(i) for i in ids) > 2, ids
    assert any(set(a) - set(b) for a, b in zip(ids, ids[1:])), f'no purge: {ids}'
    assert all(ranks[r]['ids'] == plain['ids'] for r in range(world))
    steps = [(ps, [ranks[r]['sensory'][t] for r in range(world)]) for t, ps in enumerate(plain['sensory'])]
    assert [ps['ids'] for ps, _ in steps] == plain['ids']
    # From the second detection on, the merged mask is cut from an argmax of propagated probabilities: a pixel whose two best
    # channels are closer than the cores' difference flips, and with it the mask, the values and the sensory rows.  So
    # the numbers are compared up to the first propagated frame, and afterwards who holds what.
    worst, _, _ = _check_sensory(steps[:2], world)
    _, moved, idle = _check_sensory([({'ids': ps['ids'], 'block': torch.zeros(len(ps['ids']), 1)},
                                      [dict(s, block=None if s['block'] is None else torch.zeros(len(s['ids']), 1))
                                       for s in rs]) for ps, rs in steps], world)
    assert moved >= 1, f'the survivors of the purge did not change rank: {ids}'
    _report(f'world {world} detections (ids {ids}; {moved} rows changed rank, {idle} rank-steps without objects): sensory '
            f'rows vs plain core up to the first propagated frame, relative', worst, SENSORY_REL)
    assert worst < SENSORY_REL
    _check_probs(f'world {world} detections, first two frames', ranks, plain, PROB_DET, upto=2)
    flips = max(float(((a - b).abs() > 0.5).float().mean()) for a, b in zip(ranks[0]['probs'], plain['probs']))
    _report(f'world {world} detections + purge: share of pixels on another side of a merged mask than in the plain core',
            flips, 0.02)
    assert flips < 0.02


@gpu
@pytest.mark.parametrize('world', (2, 4))
def test_real_size_session_matches_plain_core(world, golden_dir, tmp_path_factory):
    """480 x 864 (1620 tokens per frame), 5 objects, 8 frames: shards longer than top_k, production tile schedules, three
    consolidations and two evictions with the global threshold."""
    from deva.inference.sharded_core import token_bounds
    ranks = [r['real'] for r in _ranks(world, golden_dir, tmp_path_factory)]
    _, meta = _clip(golden_dir)
    cfg = dict(meta['config'], **REAL_CFG)
    plain = _plain('real', cfg, lambda core: _run_real(core, 'cuda'))
    hw = REAL_H // 16 * (REAL_W // 16)
    longs = [s['0'][1] for s in plain['sizes']]
    assert plain['sizes'][0]['0'] == [hw, 0]
    assert longs[3] == 128 and 128 < longs[5] < 256 and longs[7] <= 240, f'consolidations / evictions: {longs}'
    for t, s in enumerate(plain['sizes']):
        w, l = s['0']
        for r in range(world):
            t0, t1 = token_bounds(hw, world, r)
            assert ranks[r]['sizes'][t]['0'][0] == w // hw * (t1 - t0)
        got = [ranks[r]['sizes'][t]['0'][1] for r in range(world)]
        assert sum(got) == l, f'frame {t}: ranks hold {got} long-term slots, the plain bank {l}'
    print(f'[sharded-ranks] world {world} 480x864: plain long-term sizes {longs}, per rank at the end '
          f'{[ranks[r]["sizes"][-1]["0"][1] for r in range(world)]}')
    _check_probs(f'world {world} 480x864, 5 objects', ranks, plain, PROB_REAL)
