"""BURST's per-segment COCO RLE encoded on the device (deva/utils/rle_encode.py) against the host path: the kernels and
the result saver.

    python tools/bench_rle.py [--iters 20] [--host-iters 3] [--frames 10]

  * kernel: CUDA-event time of deva_b200_rle_encode over repeated encodes with the int64 id map resident, on ellipse
    id maps (bench_png.ellipse_ids) at 720p and 1080p with K = 10, 50 and 200 seg ids, and on a 1080p salt-and-pepper
    map (a random id in {0, 1, 2} at every pixel, seg ids 1 and 2), next to the host path on the same map: per segment
    ``ids == id``, ``np.asfortranarray`` and ``pycocotools.mask.encode``, timed with pycocotools only when it imports.
    Without it the row says ``"pycocotools": "not installed"`` and ``host_ms`` is the compare and the copy alone;
  * per_frame_1080p: this package's ResultSaver in burst mode with rle_encoder='pycocotools' and 'device' (the index PNG
    encoded on the device in both, so that the rows differ by the RLE alone), prob float32 [K+1, 480, 854] ->
    save_mask(need_resize=True, shape=(1080, 1920)) for K in 10, 50, 200: ``save_ms`` (host time of a save_mask call
    while the queue has room) and ``writer_ms`` (the writer thread's busy time per frame), as tools/bench_saver.py
    measures them.  Without pycocotools the host row runs with an encode that returns an empty string, so its
    writer_ms is the download's wait, the compares and the copies alone, and it says so;
  * bytes per frame each path moves for the RLE: the host path downloads the int64 id map; the device path uploads the
    seg ids and downloads the offsets and the strings' first min(PREFIX, bound) bytes (the rest only when longer).
Prints one JSON line with the card and its power limit read in the same run."""
import argparse
import importlib
import json
import os
import shutil
import sys
import tempfile
import time
import types

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_saver as bs  # noqa: E402  (puts the package and bench on sys.path)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_ingest import card  # noqa: E402
from bench_png import ellipse_ids  # noqa: E402


def pycocotools_mask():
    try:
        return importlib.import_module('pycocotools.mask')
    except ImportError:
        return None


def maps():
    out = {}
    for h, w, name in ((720, 1280, '720p'), (1080, 1920, '1080p')):
        for k in (10, 50, 200):
            out[f'{name}_ellipses_k{k}'] = (ellipse_ids(h, w, k).astype(np.int64), list(range(1, k + 1)))
    noise = np.random.default_rng(0).integers(0, 3, (1080, 1920)).astype(np.int64)
    out['1080p_salt_and_pepper_k2'] = (noise, [1, 2])
    return out


def host_ms(ids, seg, mask_util, iters):
    times = []
    for _ in range(iters):
        t0 = time.perf_counter()
        for i in seg:
            m = np.asfortranarray(ids == i)
            if mask_util is not None:
                mask_util.encode(m)
        times.append(time.perf_counter() - t0)
    return min(times) * 1e3


def kernel(iters, host_iters):
    from deva import _native
    from deva.utils.rle_encode import PREFIX, encode_rle
    mask_util = pycocotools_mask()
    out = {}
    for name, (ids, seg) in maps().items():
        h, w = ids.shape
        n = len(seg)
        dev = torch.from_numpy(ids).cuda()
        seg_dev = torch.tensor(seg, dtype=torch.int64, device='cuda')
        bound = _native.rle_bound(h, w, n)
        buf = torch.empty(bound, dtype=torch.uint8, device='cuda')
        ws = torch.empty(_native.rle_workspace_bytes(h, w, n), dtype=torch.uint8, device='cuda')
        offsets = torch.empty(n + 1, dtype=torch.int64, device='cuda')
        for _ in range(3):
            _native.rle_encode(dev, seg_dev, ws, buf, offsets)
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(iters):
            _native.rle_encode(dev, seg_dev, ws, buf, offsets)
        end.record()
        end.synchronize()
        strings = sum(len(r['counts']) for r in encode_rle(dev, seg))
        row = {'kernel_ms': round(start.elapsed_time(end) / iters, 4),
               'host_ms': round(host_ms(ids, seg, mask_util, host_iters), 2), 'string_bytes': strings,
               'host_download_bytes': h * w * 8,
               'device_upload_bytes': 8 * n, 'device_download_bytes': 8 * (n + 1) + min(PREFIX, bound) +
               max(0, strings - PREFIX), 'device_buffer_bytes': bound + int(ws.numel())}
        if mask_util is None:
            row['pycocotools'] = 'not installed'
        out[name] = row
    return out


def per_frame(n):
    import deva.inference.result_utils as ru
    ru.Queue = bs.TimedQueue  # only the frame queue calls task_done(), so only it accumulates
    mask_util = pycocotools_mask()
    if mask_util is None:  # the host leg's encode returns an empty string: its time is the compares and copies
        stub = types.ModuleType('pycocotools')
        stub.mask = types.ModuleType('pycocotools.mask')
        stub.mask.encode = lambda m: {'size': list(m.shape), 'counts': b''}
        sys.modules['pycocotools'], sys.modules['pycocotools.mask'] = stub, stub.mask
    g = torch.Generator(device='cuda').manual_seed(0)
    rows = {}
    for k in (10, 50, 200):
        prob = torch.softmax(4 * torch.randn(k + 1, 480 // 8, 854 // 8, device='cuda', generator=g), 0)
        prob = torch.nn.functional.interpolate(prob[None], (480, 854), mode='bilinear')[0].contiguous()
        for enc in ('pycocotools', 'device'):
            root = tempfile.mkdtemp()
            try:
                saver = ru.ResultSaver(root, 'ds/v', dataset='burst', object_manager=bs.make_om(k, False),
                                       png_encoder='device', rle_encoder=enc)
                kw = dict(need_resize=True, shape=(1080, 1920))
                for i in range(ru.RING_SIZE + 1):  # first use: kernels, every pinned slot
                    saver.save_mask(prob, f'warm{i}.jpg', **kw)
                saver.queue.join()
                saver.queue.busy, saver.queue.items = 0.0, 0
                torch.cuda.synchronize()
                calls = []
                t0 = time.perf_counter()
                for i in range(n):
                    a = time.perf_counter()
                    saver.save_mask(prob, f'{i:05d}.jpg', **kw)
                    calls.append(time.perf_counter() - a)
                saver.end()
                wall = time.perf_counter() - t0
                free = calls[:ru.QUEUE_SIZE - 1]  # later calls wait for the writer (back-pressure)
                row = {'save_ms': round(sum(free) * 1e3 / len(free), 3),
                       'writer_ms': round(saver.queue.busy * 1e3 / saver.queue.items, 2),
                       'wall_ms_per_frame': round(wall * 1e3 / n, 2), 'frames': n,
                       'segments': len(saver.all_annotations[-1]['segmentations'])}
                if enc == 'pycocotools' and mask_util is None:
                    row['pycocotools'] = 'not installed: encode returns an empty string'
                rows[f'k{k}_{enc}'] = row
            finally:
                shutil.rmtree(root, ignore_errors=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--host-iters', type=int, default=3)
    ap.add_argument('--frames', type=int, default=10)
    args = ap.parse_args()
    from deva import _native
    _native.require_device()
    torch.set_grad_enabled(False)
    out = {'card': card(), 'cpu_threads': torch.get_num_threads(), 'kernel': kernel(args.iters, args.host_iters),
           'per_frame_1080p': per_frame(args.frames)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
