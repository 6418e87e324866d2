"""Overlay JPEG encoding on the device (deva/utils/jpeg_encode.py) against Pillow: the kernels, the result saver and the
demo loop.

    python tools/bench_jpeg.py [--iters 20] [--frames 20] [--e2e-steps 60]

  * kernel: CUDA-event time of deva_b200_jpeg_encode on 1080p and 4K overlays (a smooth natural-looking frame blended
    with the colours of K = 16 and 50 ellipse ids, as the saver blends them), next to Pillow's encode of the same image
    on the host; both file sizes, and whether the files are equal;
  * per_frame_1080p: this package's ResultSaver in demo mode (RGB id PNG, JSON, overlay JPEG), prob float32
    [K+1, 480, 854] -> save_mask(need_resize=True, shape=(1080, 1920)) for K in 16, 50, 200 with PNG / JPEG encoders
    pil/pil, device/pil and device/device: ``save_ms`` (host time of a save_mask call while the queue has room) and
    ``writer_ms`` (the writer thread's busy time per frame), as tools/bench_saver.py measures them;
  * e2e: bench_saver's demo loop (1080p frames, c2 step at 480p, save_mask in demo mode) in frames/s with no saver and
    with each encoder pair.
Prints one JSON line with the card and its power limit read in the same run."""
import argparse
import functools
import io
import json
import os
import shutil
import sys
import tempfile
import time

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_saver as bs  # noqa: E402  (puts the package and bench on sys.path)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_ingest import card  # noqa: E402
from bench_png import ellipse_ids  # noqa: E402

PAIRS = (('pil', 'pil'), ('device', 'pil'), ('device', 'device'))  # (png_encoder, jpeg_encoder)


def frame(h, w, seed=0):
    """A smooth uint8 RGB frame: low-frequency colour waves with a little grain."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:h, :w].astype(np.float32)
    out = np.empty((h, w, 3), np.float32)
    for c in range(3):
        fy, fx, ph = rng.uniform(1, 4) / h, rng.uniform(1, 4) / w, rng.uniform(0, 6.3)
        out[..., c] = 128 + 90 * np.sin(2 * np.pi * (fy * yy + fx * xx) + ph)
    out += rng.normal(0, 4, out.shape)
    return np.clip(out, 0, 255).astype(np.uint8)


def overlay(h, w, k):
    ids = ellipse_ids(h, w, k)
    colours = np.random.default_rng(1).integers(0, 256, (k + 1, 3)).astype(np.float32)
    alpha = (ids == 0).astype(np.float32)[:, :, None] * 0.5 + 0.5
    return (frame(h, w) * alpha + colours[ids] * (1 - alpha)).astype(np.uint8)


def kernel(iters):
    from PIL import Image
    from deva import _native
    from deva.utils.jpeg_encode import encode_jpeg, quant_tables
    tables = quant_tables(75)
    out = {}
    for h, w, name in ((1080, 1920, '1080p'), (2160, 3840, '4k')):
        for k in (16, 50):
            img = overlay(h, w, k)
            dev = torch.from_numpy(img).cuda()
            buf = torch.empty(_native.jpeg_bound(h, w), dtype=torch.uint8, device='cuda')
            ws = torch.empty(_native.jpeg_workspace_bytes(h, w), dtype=torch.uint8, device='cuda')
            n = torch.empty(1, dtype=torch.int64, device='cuda')
            for _ in range(3):
                _native.jpeg_encode(dev, tables, ws, buf, n)
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(iters):
                _native.jpeg_encode(dev, tables, ws, buf, n)
            end.record()
            end.synchronize()
            ours = encode_jpeg(dev)
            pil = Image.fromarray(img)
            times = []
            for _ in range(3):
                b = io.BytesIO()
                t0 = time.perf_counter()
                pil.save(b, 'JPEG')
                times.append(time.perf_counter() - t0)
            out[f'{name}_k{k}'] = {'kernel_ms': round(start.elapsed_time(end) / iters, 4),
                                   'pil_encode_ms': round(min(times) * 1e3, 2), 'device_bytes': len(ours),
                                   'pil_bytes': len(b.getvalue()), 'equal': ours == b.getvalue()}
    return out


def per_frame(n):
    import deva.inference.result_utils as ru
    ru.Queue = bs.TimedQueue  # only the frame queue calls task_done(), so only it accumulates
    g = torch.Generator(device='cuda').manual_seed(0)
    image = frame(1080, 1920)
    rows = {}
    for k in (16, 50, 200):
        prob = torch.softmax(4 * torch.randn(k + 1, 480 // 8, 854 // 8, device='cuda', generator=g), 0)
        prob = torch.nn.functional.interpolate(prob[None], (480, 854), mode='bilinear')[0].contiguous()
        for png, jpg in PAIRS:
            root = tempfile.mkdtemp()
            try:
                saver = ru.ResultSaver(root, 'v', dataset='demo', object_manager=bs.make_om(k, True),
                                       png_encoder=png, jpeg_encoder=jpg)
                kw = dict(need_resize=True, shape=(1080, 1920), image_np=image)
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
                jpg_bytes = os.path.getsize(os.path.join(root, 'Visualizations', 'v', '00000.jpg'))
                rows[f'k{k}_{png}_{jpg}'] = {'save_ms': round(sum(free) * 1e3 / len(free), 3),
                                             'writer_ms': round(saver.queue.busy * 1e3 / saver.queue.items, 2),
                                             'wall_ms_per_frame': round(wall * 1e3 / n, 2), 'jpg_bytes': jpg_bytes,
                                             'frames': n}
            finally:
                shutil.rmtree(root, ignore_errors=True)
    return rows


def e2e(steps):
    import deva.inference.result_utils as ru
    ru.Queue = bs.TimedQueue
    savers = {f'{png}_{jpg}': functools.partial(ru.ResultSaver, png_encoder=png, jpeg_encoder=jpg)
              for png, jpg in PAIRS}
    return bs.e2e(savers, steps, steps, impls=('none', ) + tuple(savers))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--frames', type=int, default=20)
    ap.add_argument('--e2e-steps', type=int, default=60)
    args = ap.parse_args()
    from deva import _native
    _native.require_device()
    torch.set_grad_enabled(False)
    out = {'card': card(), 'cpu_threads': torch.get_num_threads(), 'kernel': kernel(args.iters),
           'per_frame_1080p': per_frame(args.frames), 'e2e_demo_1080p_in_480p_work': e2e(args.e2e_steps)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
