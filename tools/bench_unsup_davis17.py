"""Unsupervised DAVIS 2017 post-processing (``limit_max_id``) - the reference's and this package's.

    python tools/bench_unsup_davis17.py [--videos 4] [--max-objects 20] [--seed 0]

Input: a seeded synthetic set shaped like DAVIS 2017 unsupervised outputs, written to a temporary directory that is
removed afterwards: 480x854 RGB long-id PNGs (what the result saver writes), videos of 50-100 frames, 20-60 labels per
frame drawn from a per-video pool as moving rectangles.

Reference: the unmodified ``limit_max_id`` staged under oracle/_ref (oracle/build_ref.py stages deva/inference and
deva/utils), loaded by path.  Ours: ``deva.inference.postprocess_unsup_davis17.limit_max_id``.  Each writes into its own
directory; the two trees are compared file by file (mode, palette, pixels) in the same run.  Then the parts of our pass:
PNG decode on the thread pool, and the kernels alone (every frame's ``label_areas`` and ``label_to_index``, CUDA events,
frames resident).  Prints one JSON line with the card and its power limit read in the same run."""
import argparse
import importlib.util
import json
import os
import shutil
import sys
import tempfile
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, 'oracle', '_ref')
sys.path.insert(0, ROOT)
import bench  # noqa: E402,F401  (puts the package on sys.path)
sys.path.append(REF)  # after the package: only what the package lacks (deva.utils.palette) resolves there
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

import unsup_davis_scenario as us  # noqa: E402
from bench_ingest import card  # noqa: E402

H, W = 480, 854


def load_reference():
    file = os.path.join(REF, 'deva', 'inference', 'postprocess_unsup_davis17.py')
    if not os.path.isfile(file):
        raise RuntimeError('oracle/_ref/deva/inference is not staged: run python oracle/build_ref.py in the build '
                           'container')
    spec = importlib.util.spec_from_file_location('ref_postprocess_unsup_davis17', file)  # not deva.*: ours
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def make_dataset(root, videos, seed):
    """-> number of frames written."""
    rng = np.random.default_rng(seed)
    n_frames = 0
    for v in range(videos):
        t_len = int(rng.integers(50, 101))
        pool = rng.choice(np.arange(1, 1 << 24), size=80, replace=False)
        k = int(rng.integers(20, 61))  # labels per frame
        labels = rng.choice(pool, size=k, replace=False)
        boxes = np.stack([rng.integers(0, H - 40, k), rng.integers(0, W - 40, k), rng.integers(20, 160, k),
                          rng.integers(20, 200, k)], 1)
        speed = rng.integers(-3, 4, (k, 2))
        os.makedirs(os.path.join(root, f'video{v:02d}'))
        for t in range(t_len):
            lab = np.zeros((H, W), np.int64)
            for (y, x, hh, ww), (dy, dx), label in zip(boxes, speed, labels):
                y0, x0 = (y + dy * t) % (H - 20), (x + dx * t) % (W - 20)
                lab[y0:y0 + hh, x0:x0 + ww] = label
            rgb = np.stack([(lab >> 16) & 255, (lab >> 8) & 255, lab & 255], -1).astype(np.uint8)
            Image.fromarray(rgb).save(os.path.join(root, f'video{v:02d}', f'{t:05d}.png'))
        n_frames += t_len
    return n_frames


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def parts(src, max_num_objects):
    """Decode of every frame on the thread pool, then the kernels over the resident frames."""
    from deva import _native as nat
    from deva.inference import postprocess_unsup_davis17 as pp
    from deva.utils.png_pipeline import Decoder, Uploader
    dec = Decoder(pp.read_frame)
    videos = sorted(os.listdir(src))
    t0 = time.perf_counter()
    decoded = [list(dec.frames([os.path.join(src, v, f) for f in sorted(os.listdir(os.path.join(src, v)))]))
               for v in videos]
    decode_s = time.perf_counter() - t0
    threads = dec.pool._max_workers
    dec.close()
    upload = Uploader(torch.device('cuda'))
    on_dev = [[upload(a) for a in frames] for frames in decoded]
    tables = []
    for frames in on_dev:
        existing, _ = pp.select_objects(pp._label_lists(frames, frames[0].device), max_num_objects)
        tables.append([torch.from_numpy(a).cuda() for a in pp.index_table(existing)])
    n = sum(len(f) for f in on_dev)
    buf = torch.empty(n, 2 * pp.CAPACITY + 2, dtype=torch.int32, device='cuda')
    out = torch.empty(H, W, dtype=torch.uint8, device='cuda')

    def areas():
        i = 0
        for frames in on_dev:
            for f in frames:
                nat.label_areas(f, buf[i, :pp.CAPACITY], buf[i, pp.CAPACITY:2 * pp.CAPACITY], buf[i, 2 * pp.CAPACITY:])
                i += 1

    def rewrite():
        for frames, (labels, index) in zip(on_dev, tables):
            for f in frames:
                nat.label_to_index(f, labels, index, out)

    res = {}
    for name, fn in (('label_areas', areas), ('label_to_index', rewrite)):
        fn()
        reps = 5
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res[name] = e0.elapsed_time(e1) / reps / n
    return {'decode_ms': round(decode_s * 1e3 / n, 3), 'label_areas_kernel_ms': round(res['label_areas'], 4),
            'label_to_index_kernel_ms': round(res['label_to_index'], 4), 'decode_threads': threads}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--videos', type=int, default=4)
    ap.add_argument('--max-objects', type=int, default=20)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--png-decoder', choices=('pil', 'device', 'both'), default='pil',
                    help="the input decoder of limit_max_id; 'both' times the two, alternating, in one run")
    args = ap.parse_args()
    decoders = ('pil', 'device') if args.png_decoder == 'both' else (args.png_decoder,)
    from deva import _native as nat
    nat.require_device()
    ref = load_reference()
    from deva.inference.postprocess_unsup_davis17 import limit_max_id
    from deva.utils.palette import davis_palette
    root = tempfile.mkdtemp()
    try:
        src = os.path.join(root, 'in')
        n = make_dataset(src, args.videos, args.seed)
        m = args.max_objects
        for d in decoders:  # CUDA context, module load, pinned pool
            limit_max_id(src, os.path.join(root, 'warm'), m, png_decoder=d)
        runs = {d: [] for d in decoders}
        for _ in range(2 if len(decoders) > 1 else 1):  # alternating, so both paths see the same machine state
            for d in decoders:
                runs[d].append(timed(lambda: limit_max_id(src, os.path.join(root, 'ours_' + d), m, png_decoder=d)))
        t = {f'ours_{d}': min(v) for d, v in runs.items()}
        t['reference'] = timed(lambda: ref.limit_max_id(src, os.path.join(root, 'ref'), m))
        want = us.snapshot(os.path.join(root, 'ref'))
        equal, davis = {}, True
        for d in decoders:
            ours = us.snapshot(os.path.join(root, 'ours_' + d))
            equal[d] = sorted(ours) == sorted(want) and all(
                ours[k][:2] == want[k][:2] and np.array_equal(ours[k][2], want[k][2]) for k in want)
            davis = davis and all(v[1] == us.sha(bytes(davis_palette)) for v in ours.values())
        out = {'card': card(), 'cpu_threads': os.cpu_count(),
               'dataset': {'videos': args.videos, 'frames': n, 'size': [H, W], 'labels_per_frame': [20, 60],
                           'max_num_objects': m},
               'per_frame_ms': {k: round(v * 1e3 / n, 3) for k, v in t.items()},
               'speedup': {d: round(t['reference'] / t['ours_' + d], 1) for d in decoders},
               'files_equal': {d: bool(v) for d, v in equal.items()}, 'files': len(want), 'palette_is_davis': davis,
               'ours_parts_per_frame': parts(src, m)}
        print(json.dumps(out))
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == '__main__':
    main()
