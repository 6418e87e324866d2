"""Device JPEG decode (csrc/jpeg_decode.cu, deva/utils/jpeg_decode.py) against Pillow.

For overlay frames written by Pillow at 480p, 720p, 1080p and 4K, at quality 75 and 95, 4:2:0 and 4:4:4, reports:
  * the kernel time per file from CUDA events with the inputs resident on the device, for one file alone and per file
    of an 8-file batch, and the synchronisation rounds the entropy decode took;
  * each kernel's share, from a torch.profiler run of its own, and the host time of ``parse``;
  * Pillow's decode of the same files on one host thread and on all of them.
Prints one JSON line with the card and its power limit read in the same run."""
import argparse
import io
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402,F401  (puts the package on sys.path)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

import jpeg_cases as jc  # noqa: E402
from bench_ingest import card  # noqa: E402

SIZES = {'480p': (480, 854), '720p': (720, 1280), '1080p': (1080, 1920), '4K': (2160, 3840)}
BATCH = 8


def files(h, w, q, ss, n):
    out = []
    for t in range(n):
        b = io.BytesIO()
        Image.fromarray(jc.overlay(h, w, seed=t)).save(b, 'JPEG', quality=q, subsampling=ss)
        out.append(b.getvalue())
    return out


def kernel_ms(datas, iters):
    from deva import _native
    from deva.utils import jpeg_decode as jd
    args, arrays = jd.stage([jd.parse(d) for d in datas])
    for _ in range(3):
        _native.jpeg_decode(*args)
    torch.cuda.synchronize()
    assert args[7].tolist() == [0] * len(datas)
    for d, a in zip(datas, arrays):
        assert np.array_equal(a.cpu().numpy(), np.asarray(Image.open(io.BytesIO(d))))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        _native.jpeg_decode(*args)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters / len(datas), jd.sync_rounds(args)


def stage_ms(datas, iters):
    from deva import _native
    from deva.utils import jpeg_decode as jd
    args, _ = jd.stage([jd.parse(d) for d in datas])
    _native.jpeg_decode(*args)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            _native.jpeg_decode(*args)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        name = ev.key.split('(')[0].split('::')[-1]
        if 'kernel' in name:
            out[name] = round(ev.device_time_total / 1e3 / iters / len(datas), 4)
    return out


def parse_ms(datas):
    """Host time of ``parse`` per file: the marker walk, table build, unstuffing and interval cut."""
    from deva.utils import jpeg_decode as jd
    t = time.perf_counter()
    for d in datas:
        jd.parse(d)
    return round((time.perf_counter() - t) * 1e3 / len(datas), 3)


def pillow_ms(datas, threads):
    def one(d):
        return np.asarray(Image.open(io.BytesIO(d)))
    with ThreadPoolExecutor(threads) as pool:
        list(pool.map(one, datas))
        t = time.perf_counter()
        for _ in range(3):
            list(pool.map(one, datas))
    return (time.perf_counter() - t) * 1e3 / 3 / len(datas)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='480p,720p,1080p,4K')
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    torch.cuda.init()
    rows = []
    threads = os.cpu_count() or 1
    for size in a.sizes.split(','):
        h, w = SIZES[size]
        for q in (75, 95):
            for ss in (2, 0):
                datas = files(h, w, q, ss, BATCH)
                alone, rounds = kernel_ms(datas[:1], a.iters)
                batch, rounds_b = kernel_ms(datas, a.iters)
                row = dict(size=size, quality=q, sampling='4:2:0' if ss == 2 else '4:4:4',
                           kb=round(sum(map(len, datas)) / len(datas) / 1024, 1),
                           alone_ms=round(alone, 4), batch_ms_per_file=round(batch, 4), rounds_alone=rounds,
                           rounds_batch=rounds_b, stages_ms_per_file=stage_ms(datas, 5), parse_ms=parse_ms(datas),
                           pillow_1_thread_ms=round(pillow_ms(datas, 1), 3),
                           pillow_all_threads_ms=round(pillow_ms(datas, threads), 3))
                print(json.dumps(row), flush=True)
                rows.append(row)
    result = dict(card=card(), host_threads=threads, rows=rows)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_jpeg_decode.json'), 'w') as f:
            json.dump(result, f, indent=1)
    print(json.dumps(dict(card=result['card'], host_threads=threads)))


if __name__ == '__main__':
    main()
