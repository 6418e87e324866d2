"""Time one MemoryManager.match_memory read at the c2 and c3 read shapes for a range of top_k, and one full
DEVAInferenceCore.step at c3 for top_k 30 and 64 (CUDA events, after warm-up).

    python tools/bench_topk.py [--reps 20] [--out bench_topk.json]

c2: q = 1620 query pixels (a 480 x 864 frame at 1/16) against a 2000-slot window; c3: q = 8160 (1080 x 1920) against
10 000 slots; two objects of 128 value channels.  top_k <= 32 takes sim_topk's fused path, top_k > 32 the wide path
(dense similarity row + radix select).  Prints the card name and power limit read in the same process, and one line per
case; writes the table as JSON when --out is given.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, 'tracking-anything-with-deva_b200')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

CK, CV = 64, 128
READS = {'c2': (30, 54, 2000), 'c3': (68, 120, 10000)}   # query h, w at 1/16 and window slots
TOP_KS = (30, 32, 33, 50, 64, 100, 128, 256)


def _card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else 'unknown'


def _manager(top_k):
    from deva.inference.memory_manager import MemoryManager
    cfg = dict(key_dim=CK, value_dim=512, pix_feat_dim=512, mem_every=1, enable_long_term=True, chunk_size=-1,
               top_k=top_k, enable_long_term_count_usage=True, max_mid_term_frames=10, min_mid_term_frames=5,
               num_prototypes=128, max_long_term_elements=10000)
    return MemoryManager(cfg)


def _timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def time_read(shape, top_k, reps):
    h, w, n = READS[shape]
    g = torch.Generator(device='cuda').manual_seed(0)
    mgr = _manager(top_k)
    # one append of n slots (a memory frame of n tokens), then the read of an h x w query
    key = torch.randn(1, CK, 1, n, generator=g, device='cuda')
    shr = 1 + torch.rand(1, 1, 1, n, generator=g, device='cuda')
    sel = torch.sigmoid(torch.randn(1, CK, 1, n, generator=g, device='cuda'))
    val = torch.randn(1, 2, CV, 1, n, generator=g, device='cuda')
    mgr.add_memory(key, shr, val, [1, 2], selection=sel)
    qk = torch.randn(1, CK, h, w, generator=g, device='cuda')
    qe = torch.sigmoid(torch.randn(1, CK, h, w, generator=g, device='cuda'))
    return _timed(lambda: mgr.match_memory(qk, qe), reps)


def time_step(top_k, reps):
    from deva.inference.inference_core import DEVAInferenceCore
    from deva.model.network import DEVA
    from deva.model.param_spec import synthetic_state_dict
    cfg = dict(key_dim=CK, value_dim=512, pix_feat_dim=512, mem_every=5, enable_long_term=True, chunk_size=-1,
               top_k=top_k, enable_long_term_count_usage=True, max_mid_term_frames=10, min_mid_term_frames=5,
               num_prototypes=128, max_long_term_elements=10000)
    net = DEVA(cfg).cuda().eval()
    net.load_weights({k: v.cuda() for k, v in synthetic_state_dict(seed=1).items()})
    core = DEVAInferenceCore(net, cfg)
    g = torch.Generator(device='cuda').manual_seed(1)
    H, W = 1088, 1920
    img = torch.randn(3, H, W, generator=g, device='cuda')
    mask = torch.zeros(H, W, dtype=torch.long, device='cuda')
    mask[100:500, 100:700] = 1
    mask[500:1000, 900:1700] = 2
    core.step(img, mask, [1, 2])
    for _ in range(4):   # a few memory frames (mem_every 5 keeps the bank fixed inside the timed window)
        core.step(img + 0.05 * torch.randn(3, H, W, generator=g, device='cuda'))
    frame = img + 0.05 * torch.randn(3, H, W, generator=g, device='cuda')
    return _timed(lambda: core.step(frame), reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_topk: needs a CUDA device')
    from deva import _native
    _native.require_device()
    card = _card()
    print('card, power limit:', card)
    rows = []
    for shape in READS:
        for top_k in TOP_KS:
            ms = time_read(shape, top_k, args.reps)
            rows.append(dict(case=f'match_memory {shape}', top_k=top_k, ms=ms))
            print(f'match_memory {shape} top_k {top_k:4d}: {ms:8.3f} ms')
    for top_k in (30, 64):
        ms = time_step(top_k, max(5, args.reps // 4))
        rows.append(dict(case='step c3', top_k=top_k, ms=ms))
        print(f'step c3 (1088 x 1920) top_k {top_k:4d}: {ms:8.3f} ms')
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(dict(card=card, rows=rows), open(args.out, 'w'), indent=1)


if __name__ == '__main__':
    main()
