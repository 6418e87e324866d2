"""PNG encoding on the device (deva/utils/png_encode.py) against Pillow: the kernels, the result saver and the demo loop.

    python tools/bench_png.py [--iters 20] [--frames 20] [--e2e-steps 60]

  * kernel: CUDA-event time of deva_b200_png_encode on 1080p and 4K RGB id maps and index maps (K = 16 and 50 ellipse
    objects), next to Pillow's encode of the same image on the host and both file sizes;
  * per_frame_1080p: this package's ResultSaver with png_encoder='pil' and 'device', prob float32 [K+1, 480, 854] ->
    save_mask(need_resize=True, shape=(1080, 1920)) in demo mode (RGB id PNG, JSON, overlay JPEG) and vipseg mode
    (index PNG, JSON) for K in 16, 50, 200: ``save_ms`` (host time of a save_mask call while the queue has room) and
    ``writer_ms`` (the writer thread's busy time per frame), as tools/bench_saver.py measures them;
  * e2e: bench_saver's demo loop (1080p frames, c2 step at 480p, save_mask in demo mode) in frames/s with no saver,
    with 'pil' and with 'device'.
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


def ellipse_ids(h, w, k, seed=0):
    rng = np.random.default_rng(seed)
    ids = np.zeros((h, w), np.int32)
    yy, xx = np.ogrid[:h, :w]
    for i in range(1, k + 1):
        cy, cx = rng.uniform(0, h), rng.uniform(0, w)
        ry, rx = rng.uniform(h / 20, h / 4), rng.uniform(w / 20, w / 4)
        ids[((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1] = i
    return ids


def kernel(iters):
    from PIL import Image
    from deva import _native
    from deva.utils.png_encode import encode_png, pillow_png_layout
    palette = [(37 * i) % 256 for i in range(768)]
    out = {}
    for h, w, name in ((1080, 1920, '1080p'), (2160, 3840, '4k')):
        for k in (16, 50):
            ids = ellipse_ids(h, w, k)
            lut = np.random.default_rng(1).integers(0, 256, (k + 1, 3), dtype=np.uint8)
            lut[0] = 0
            for kind, img, mode in (('rgb', lut[ids], 'RGB'), ('index', ids.astype(np.uint8), 'P')):
                dev = torch.from_numpy(np.ascontiguousarray(img)).cuda()
                channels, bits = (3 if mode == 'RGB' else 1), pillow_png_layout(mode, palette)[0]
                bound = _native.png_bound(h, w, channels, bits)
                buf = torch.empty(bound, dtype=torch.uint8, device='cuda')
                ws = torch.empty(_native.png_workspace_bytes(h), dtype=torch.uint8, device='cuda')
                n = torch.empty(1, dtype=torch.int64, device='cuda')
                for _ in range(3):
                    _native.png_encode(dev, bits, ws, buf, n)
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                for _ in range(iters):
                    _native.png_encode(dev, bits, ws, buf, n)
                end.record()
                end.synchronize()
                ours = encode_png(dev, mode, palette)
                pil = Image.fromarray(img)
                if mode == 'P':
                    pil.putpalette(palette)
                t0 = time.perf_counter()
                b = io.BytesIO()
                pil.save(b, format='PNG')
                pil_ms = (time.perf_counter() - t0) * 1e3
                out[f'{name}_{kind}_k{k}'] = {'kernel_ms': round(start.elapsed_time(end) / iters, 4),
                                              'pil_encode_ms': round(pil_ms, 2), 'device_bytes': len(ours),
                                              'pil_bytes': len(b.getvalue()), 'raw_bytes': img.nbytes}
    return out


def per_frame(n):
    import deva.inference.result_utils as ru
    ru.Queue = bs.TimedQueue  # only the frame queue calls task_done(), so only it accumulates
    g = torch.Generator(device='cuda').manual_seed(0)
    image = np.random.default_rng(0).integers(0, 256, (1080, 1920, 3), dtype=np.uint8)
    rows = {}
    for mode, long_id in (('demo', True), ('vipseg', False)):
        for k in (16, 50, 200):
            prob = torch.softmax(4 * torch.randn(k + 1, 480 // 8, 854 // 8, device='cuda', generator=g), 0)
            prob = torch.nn.functional.interpolate(prob[None], (480, 854), mode='bilinear')[0].contiguous()
            for enc in ('pil', 'device'):
                root = tempfile.mkdtemp()
                try:
                    saver = ru.ResultSaver(root, 'v', dataset=mode, object_manager=bs.make_om(k, long_id),
                                           png_encoder=enc)
                    kw = dict(need_resize=True, shape=(1080, 1920), image_np=image if mode == 'demo' else None)
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
                    rows[f'{mode}_k{k}_{enc}'] = {'save_ms': round(sum(free) * 1e3 / len(free), 3),
                                                  'writer_ms': round(saver.queue.busy * 1e3 / saver.queue.items, 2),
                                                  'wall_ms_per_frame': round(wall * 1e3 / n, 2), 'frames': n}
                finally:
                    shutil.rmtree(root, ignore_errors=True)
    return rows


def e2e(steps):
    import deva.inference.result_utils as ru
    ru.Queue = bs.TimedQueue
    savers = {enc: functools.partial(ru.ResultSaver, png_encoder=enc) for enc in ('pil', 'device')}
    return bs.e2e(savers, steps, steps, impls=('none', 'pil', 'device'))


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
