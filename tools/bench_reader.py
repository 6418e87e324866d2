"""Frames per second of the evaluation drivers' ingest: the dataset reader under DataLoader against DeviceLoader.

    python tools/bench_reader.py [--frames 64] [--size 480] [--out results/bench_reader.json]

Seeded clips are generated in a temporary directory: ``--frames`` frames at 480p, 1080p and 4K (q90 JPEG, 4:2:0) and a
P first-frame mask.  For each clip, ``VideoReader(size=--size)`` is read through
  * ``DataLoader(reader, batch_size=1, num_workers=2)``, as the drivers run it;
  * the same with ``num_workers`` equal to the host's cores;
  * ``DeviceLoader(reader)``;
each item's rgb and mask moved to the device as the drivers do (``.cuda()``), ending in a device synchronise.  Kernel
time per frame is the window's JPEG decode and resize from CUDA events.  For the 1080p and 4K clips (480x853 at size
480) an eval_vos-shaped loop runs under each loader: bench.py's c2-like ``step`` (a core whose bank is pre-filled with the
clip's five objects, so the first frame's mask and labels are read but not added again), then ``prob_to_ids`` back to
the source size and its download, with no file writes.  One JSON line, with the card, its power limit and the host's CPU
count read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (puts the package on sys.path)
import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402
from torch.utils.data import DataLoader  # noqa: E402

SOURCES = {'480p': (480, 854), '1080p': (1080, 1920), '4K': (2160, 3840)}


def card():
    try:
        return subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=name,power.limit,clocks.max.sm',
                               '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f'unavailable ({e})'


def make_clip(root, h, w, frames, seed):
    rng = np.random.default_rng(seed)
    img_dir, mask_dir = os.path.join(root, 'JPEGImages', 'clip'), os.path.join(root, 'Annotations', 'clip')
    os.makedirs(img_dir)
    os.makedirs(mask_dir)
    base = np.asarray(Image.fromarray(rng.integers(0, 256, (h // 16 + 1, w // 16 + 1, 3), dtype=np.uint8)).resize(
        (w, h), Image.BILINEAR))
    for t in range(frames):
        frame = np.roll(base, 4 * t, axis=1)
        Image.fromarray(frame).save(os.path.join(img_dir, f'{t:05d}.jpg'), quality=90, subsampling=2)
    mask = np.zeros((h, w), np.uint8)
    for o in range(1, 6):
        mask[(o * h) // 8:(o * h) // 8 + h // 6, (o * w) // 8:(o * w) // 8 + w // 6] = o
    im = Image.frombytes('P', (w, h), mask.tobytes())
    im.putpalette([v for i in range(256) for v in (i * 40 % 256, i * 80 % 256, i * 120 % 256)])
    im.save(os.path.join(mask_dir, '00000.png'))
    return img_dir, mask_dir


def drain(loader, per_item=None):
    """Seconds to iterate ``loader``, moving rgb and mask to the device as the drivers do, to a device synchronise."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 0
    for i, data in enumerate(loader):
        rgb = data['rgb'].cuda()[0]
        mask = data.get('mask')
        mask = mask.cuda()[0] if mask is not None else None
        if per_item is not None:
            per_item(i, data, rgb, mask)
        n += 1
    torch.cuda.synchronize()
    return time.perf_counter() - t0, n


def kernel_ms_per_frame(img_dir, size, window=8, reps=5):
    """CUDA-event time of one window's JPEG decode launch and its frames' resizes, per frame."""
    from deva.inference.frame_io import frame_from_rgb8
    from deva.utils import jpeg_decode
    files = sorted(os.listdir(img_dir))[:window]
    headers = [jpeg_decode.parse(open(os.path.join(img_dir, f), 'rb').read()) for f in files]
    times = []
    for r in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        status, arrays, keep = jpeg_decode.enqueue(headers)  # noqa: F841
        outs = [frame_from_rgb8(x, size=size) for x in arrays]  # noqa: F841  (alive until the timing ends)
        b.record()
        torch.cuda.synchronize()
        assert status.eq(0).all(), status
        if r:
            times.append(a.elapsed_time(b) / len(files))
    return round(float(np.median(times)), 3)


def eval_loop(loader_fn, wl_w, size):
    """fps of an eval_vos-shaped loop: step on each frame, prob_to_ids to the source size."""
    from deva.inference.frame_io import prob_to_ids
    wl = dict(bench.WORKLOADS['c2'], w=wl_w)
    clip = bench.Clip(wl, torch.device('cuda', 0), seed=0)

    def per_item(i, data, rgb, mask):
        assert tuple(rgb.shape[1:]) == (wl['h'], wl['w']), rgb.shape
        if mask is not None:  # read as the driver does; the pre-filled core already holds the clip's objects
            data['valid_labels'].tolist()
        p = clip.core.step(rgb)
        shape = tuple(int(v) for v in data['info']['shape'])
        prob_to_ids(p, clip.core.object_manager, size=shape, dtype=torch.uint8).cpu()
        clip.clamp()
    secs, n = drain(loader_fn(), per_item)
    return round(n / secs, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=64)
    ap.add_argument('--size', type=int, default=480)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from deva import _native
    from deva.inference.data.device_loader import DeviceLoader
    from deva.inference.data.video_reader import VideoReader
    from deva.inference.frame_io import reader_size
    _native.require_device()
    torch.cuda.set_device(0)
    cores = os.cpu_count()
    result = {'card': card(), 'host_cpus': cores, 'frames': args.frames, 'size': args.size, 'clips': {}}
    with tempfile.TemporaryDirectory() as tmp:
        for k, (name, (h, w)) in enumerate(SOURCES.items()):
            img_dir, mask_dir = make_clip(os.path.join(tmp, name), h, w, args.frames, k)

            def reader():
                return VideoReader('clip', img_dir, mask_dir, size=args.size)
            loaders = {'dataloader_2_workers': lambda: DataLoader(reader(), batch_size=1, num_workers=2),
                       f'dataloader_{cores}_workers': lambda: DataLoader(reader(), batch_size=1, num_workers=cores),
                       'device_loader': lambda: DeviceLoader(reader())}
            drain(DeviceLoader(reader()))  # warm-up: module load, tables, allocator
            res = {}
            for lname, fn in loaders.items():
                secs, n = drain(fn())
                res[f'{lname}_fps'] = round(n / secs, 2)
            res['kernel_ms_per_frame'] = kernel_ms_per_frame(img_dir, args.size)
            oh, ow = reader_size(h, w, args.size)
            if (oh, ow) == (480, 853):  # bench.py's c2 working size
                for lname, fn in loaders.items():
                    res[f'eval_loop_{lname}_fps'] = eval_loop(fn, ow, args.size)
            result['clips'][name] = res
            print(name, res, flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or '.', exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
