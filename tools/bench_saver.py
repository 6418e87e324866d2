"""Per-frame cost of the result saver, the reference's and this package's, and one end-to-end demo loop with each.

    python tools/bench_saver.py [--frames 20] [--ref-frames 4] [--e2e-steps 60] [--ref-e2e-steps 15] [--path-to-image]

Per frame at 1080p: prob float32 [K+1, 480, 854] on the device, save_mask(need_resize=True, shape=(1080, 1920)) in
  * demo mode (long ids: RGB id PNG, JSON areas, overlay JPEG from a uint8 image_np) and
  * vipseg mode (uint8 index PNG, JSON areas),
for K in 16, 50, 200.  ``save_ms`` is the host time of a save_mask call while the queue has room; ``writer_ms`` is the saver thread's busy time
per frame (queue.get to task_done: remap, areas, colouring, blending, encoding, file writes; for this package also the
wait on the frame's copies).  Files go to a temporary directory that is removed afterwards.

End to end: 1080p uint8 host frames -> frame_from_rgb8(size=480) -> step (bench.py's c2 setup: 5 objects, 2k slots,
at 480x853) -> save_mask(need_resize=True, shape=(1080, 1920), image_np=frame) in demo mode with long ids, then end();
frames/s over the whole run, next to the same loop without a saver.

With --path-to-image, only the overlay given as a file is measured, with this package's saver and both device encoders:
the demo frames are 1080p JPEGs (Pillow quality 90, 4:2:0) passed as path_to_image, decoded by Pillow on the writer
thread and blended on the host (jpeg_decoder='pil') or decoded and blended on the device (jpeg_decoder='device').  It
reports save_ms / writer_ms per frame for K = 16 and the end-to-end loop with each decoder, next to the same loop with
the frames as image_np.

The reference's ResultSaver is the unmodified module staged under oracle/_ref (oracle/build_ref.py), loaded by path
under its own module name; oracle/_ref goes on sys.path after this package, so its imports of deva.* resolve to this
package first and to the staged reference for what this package lacks (deva.utils.pano_utils).  pycocotools and
supervision, which it imports eagerly and these modes never call, are stubbed when absent.  Prints one JSON line with
the card and its power limit read in the same run."""
import argparse
import importlib.util
import json
import os
import queue
import shutil
import sys
import tempfile
import time
import types

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, 'oracle', '_ref')
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (puts the package on sys.path)
sys.path.append(REF)  # after the package: only what the package lacks resolves there
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_ingest import card  # noqa: E402
from deva.inference.result_utils import QUEUE_SIZE, RING_SIZE  # noqa: E402


class TimedQueue(queue.Queue):
    """The saver's frame queue, timing the writer thread from get() to task_done()."""

    def __init__(self, maxsize=0):
        super().__init__(maxsize)
        self.busy, self.items, self._t = 0.0, 0, None

    def get(self, *a, **k):
        item = super().get(*a, **k)
        if item is not None:
            self._t = time.perf_counter()
        return item

    def task_done(self):
        if self._t is not None:
            self.busy += time.perf_counter() - self._t
            self.items += 1
            self._t = None
        super().task_done()


def load_savers():
    for name in ('pycocotools', 'supervision'):
        try:
            importlib.import_module(name)
        except ImportError:
            stub = types.ModuleType(name)
            stub.mask = types.ModuleType(name + '.mask')
            sys.modules[name], sys.modules[name + '.mask'] = stub, stub.mask
    path = os.path.join(REF, 'deva', 'inference', 'result_utils.py')
    if not os.path.isfile(path):
        raise RuntimeError('oracle/_ref is not staged: run python oracle/build_ref.py in the build container')
    spec = importlib.util.spec_from_file_location('ref_result_utils', path)  # not deva.*: that name is this package's
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    import deva.inference.result_utils as ours
    assert ref.ID2RGBConverter.__module__ == 'deva.utils.pano_utils' and ours.__file__.startswith(bench.PKG)
    ref.Queue = ours.Queue = TimedQueue  # only the frame queue calls task_done(), so only it accumulates
    return {'reference': ref.ResultSaver, 'ours': ours.ResultSaver}


def make_om(k, long_id):
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    np.random.seed(0)
    om = ObjectManager()
    om.use_long_id = long_id
    om.add_new_objects([ObjectInfo(1000 + 37 * i if long_id else i + 1, category_id=i % 3, score=0.5)
                        for i in range(k)])
    return om


def per_frame(savers, n_ours, n_ref):
    g = torch.Generator(device='cuda').manual_seed(0)
    image = np.random.default_rng(0).integers(0, 256, (1080, 1920, 3), dtype=np.uint8)
    rows = {}
    for mode, long_id in (('demo', True), ('vipseg', False)):
        for k in (16, 50, 200):
            prob = torch.softmax(4 * torch.randn(k + 1, 480 // 8, 854 // 8, device='cuda', generator=g), 0)
            prob = torch.nn.functional.interpolate(prob[None], (480, 854), mode='bilinear')[0].contiguous()
            for impl, Saver in savers.items():
                n = n_ours if impl == 'ours' else n_ref
                root = tempfile.mkdtemp()
                try:
                    saver = Saver(root, 'v', dataset=mode, object_manager=make_om(k, long_id))
                    kw = dict(need_resize=True, shape=(1080, 1920), image_np=image if mode == 'demo' else None)
                    for i in range(RING_SIZE + 1 if impl == 'ours' else 1):  # first use: kernels, every pinned slot
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
                    # the calls made while the queue still had room: later ones wait for the writer (back-pressure)
                    free = calls[:QUEUE_SIZE - 1]
                    rows[f'{mode}_k{k}_{impl}'] = {'save_ms': round(sum(free) * 1e3 / len(free), 3),
                                                   'writer_ms': round(saver.queue.busy * 1e3 / saver.queue.items, 2),
                                                   'wall_ms_per_frame': round(wall * 1e3 / n, 2), 'frames': n}
                finally:
                    shutil.rmtree(root, ignore_errors=True)
    return rows


def encode_ms(n=5):
    """PIL alone, per 1080p frame, on images this package's kernel produced for K = 16: the host work left."""
    import io
    from PIL import Image
    from deva.inference.frame_io import prob_to_segments
    g = torch.Generator(device='cuda').manual_seed(0)
    prob = torch.softmax(4 * torch.randn(17, 480 // 8, 854 // 8, device='cuda', generator=g), 0)
    prob = torch.nn.functional.interpolate(prob[None], (480, 854), mode='bilinear')[0].contiguous()
    frame = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (1080, 1920, 3), dtype=np.uint8)).cuda()
    seg = prob_to_segments(prob, make_om(16, True), (1080, 1920), rgb=True, frame=frame)
    images = {'png_rgb_ids': (seg.rgb, 'PNG'), 'jpeg_overlay': (seg.overlay, 'JPEG'),
              'png_index': (prob_to_segments(prob, make_om(16, False), (1080, 1920)).index, 'PNG')}
    out = {}
    for name, (t, fmt) in images.items():
        img = Image.fromarray(t.cpu().numpy())
        t0 = time.perf_counter()
        for _ in range(n):
            img.save(io.BytesIO(), fmt)
        out[name] = round((time.perf_counter() - t0) * 1e3 / n, 2)
    return out


def e2e(savers, steps, ref_steps, warmup=RING_SIZE + 1, impls=('none', 'ours', 'reference')):
    """impls: 'none' (no saver) and keys of savers, in the order they run; 'reference' runs ref_steps steps."""
    from deva.inference.frame_io import frame_from_rgb8
    wl = dict(bench.WORKLOADS['c2'], w=853)  # frame_from_rgb8(size=480)'s output for a 1920x1080 frame
    g = torch.Generator().manual_seed(1)
    frames = [torch.randint(0, 256, (1080, 1920, 3), generator=g, dtype=torch.uint8).pin_memory() for _ in range(5)]
    images = [f.numpy() for f in frames]
    out = {}
    for impl in impls:
        clip = bench.Clip(wl, torch.device('cuda', 0), seed=0)
        clip.core.object_manager.use_long_id = True
        n = ref_steps if impl == 'reference' else steps
        root = tempfile.mkdtemp()
        try:
            saver = None if impl == 'none' else savers[impl](root, None, dataset='demo',
                                                             object_manager=clip.core.object_manager)

            def one(i):
                p = clip.core.step(frame_from_rgb8(frames[i % 5], size=480))
                if saver is not None:
                    saver.save_mask(p, f'{i:05d}.jpg', need_resize=True, shape=(1080, 1920), image_np=images[i % 5])
                clip.clamp()

            for i in range(warmup):
                one(i)
            if saver is not None:
                saver.queue.join()
                saver.queue.busy, saver.queue.items = 0.0, 0
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(n):
                one(i)
            if saver is not None:
                saver.end()
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3 / n
            row = {'ms_per_frame': round(ms, 2), 'fps': round(1e3 / ms, 2), 'frames': n}
            if saver is not None:
                row['writer_ms'] = round(saver.queue.busy * 1e3 / saver.queue.items, 2)
            out[impl] = row
        finally:
            shutil.rmtree(root, ignore_errors=True)
    return out


def _demo_jpegs(root, n=5):
    """n 1080p demo frames as JPEG files -> (paths, the arrays Pillow decodes them to)."""
    import io
    from PIL import Image
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    import jpeg_cases
    paths, arrays = [], []
    for t in range(n):
        b = io.BytesIO()
        Image.fromarray(jpeg_cases.overlay(1080, 1920, seed=t)).save(b, 'JPEG', quality=90)
        paths.append(os.path.join(root, f'frame{t}.jpg'))
        with open(paths[-1], 'wb') as f:
            f.write(b.getvalue())
        arrays.append(np.asarray(Image.open(io.BytesIO(b.getvalue()))).copy())
    return paths, arrays


def path_to_image(n, steps, warmup=RING_SIZE + 1):
    """save_ms / writer_ms per 1080p frame (K = 16) and the end-to-end demo loop, with the overlay's frame given as a
    JPEG path (Pillow or device decoder) or as image_np; device PNG and JPEG encoders throughout."""
    from deva.inference import result_utils
    from deva.inference.frame_io import frame_from_rgb8
    from deva.inference.result_utils import ResultSaver
    result_utils.Queue = TimedQueue  # only the frame queue calls task_done(), so only it accumulates
    src = tempfile.mkdtemp()
    paths, arrays = _demo_jpegs(src)
    variants = {'image_np': ('pil', lambda i: dict(image_np=arrays[i % 5])),
                'path_pil': ('pil', lambda i: dict(path_to_image=paths[i % 5])),
                'path_device': ('device', lambda i: dict(path_to_image=paths[i % 5]))}
    out = {'per_frame_k16': {}, 'e2e': {}}
    g = torch.Generator(device='cuda').manual_seed(0)
    prob = torch.softmax(4 * torch.randn(17, 480 // 8, 854 // 8, device='cuda', generator=g), 0)
    prob = torch.nn.functional.interpolate(prob[None], (480, 854), mode='bilinear')[0].contiguous()
    wl = dict(bench.WORKLOADS['c2'], w=853)
    frames = [torch.from_numpy(a).pin_memory() for a in arrays]
    try:
        for name, (decoder, kw) in variants.items():
            root = tempfile.mkdtemp()
            try:
                saver = ResultSaver(root, 'v', dataset='demo', object_manager=make_om(16, True), png_encoder='device',
                                    jpeg_encoder='device', jpeg_decoder=decoder)
                for i in range(warmup):
                    saver.save_mask(prob, f'warm{i}.jpg', need_resize=True, shape=(1080, 1920), **kw(i))
                saver.queue.join()
                saver.queue.busy, saver.queue.items = 0.0, 0
                torch.cuda.synchronize()
                calls = []
                for i in range(n):
                    a = time.perf_counter()
                    saver.save_mask(prob, f'{i:05d}.jpg', need_resize=True, shape=(1080, 1920), **kw(i))
                    calls.append(time.perf_counter() - a)
                saver.end()
                free = calls[:QUEUE_SIZE - 1]
                out['per_frame_k16'][name] = {'save_ms': round(sum(free) * 1e3 / len(free), 3),
                                              'writer_ms': round(saver.queue.busy * 1e3 / saver.queue.items, 2)}
            finally:
                shutil.rmtree(root, ignore_errors=True)
            clip = bench.Clip(wl, torch.device('cuda', 0), seed=0)
            clip.core.object_manager.use_long_id = True
            root = tempfile.mkdtemp()
            try:
                saver = ResultSaver(root, None, dataset='demo', object_manager=clip.core.object_manager,
                                    png_encoder='device', jpeg_encoder='device', jpeg_decoder=decoder)

                def one(i):
                    p = clip.core.step(frame_from_rgb8(frames[i % 5], size=480))
                    saver.save_mask(p, f'{i:05d}.jpg', need_resize=True, shape=(1080, 1920), **kw(i))
                    clip.clamp()

                for i in range(warmup):
                    one(i)
                saver.queue.join()
                saver.queue.busy, saver.queue.items = 0.0, 0
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(steps):
                    one(i)
                saver.end()
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) * 1e3 / steps
                out['e2e'][name] = {'ms_per_frame': round(ms, 2), 'fps': round(1e3 / ms, 2), 'frames': steps,
                                    'writer_ms': round(saver.queue.busy * 1e3 / saver.queue.items, 2)}
            finally:
                shutil.rmtree(root, ignore_errors=True)
    finally:
        shutil.rmtree(src, ignore_errors=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=20)
    ap.add_argument('--ref-frames', type=int, default=4)
    ap.add_argument('--e2e-steps', type=int, default=60)
    ap.add_argument('--ref-e2e-steps', type=int, default=15)
    ap.add_argument('--path-to-image', action='store_true')
    args = ap.parse_args()
    from deva import _native as nat
    nat.require_device()
    torch.set_grad_enabled(False)
    if args.path_to_image:
        print(json.dumps({'card': card(), 'cpu_threads': torch.get_num_threads(),
                          'path_to_image_1080p_demo': path_to_image(args.frames, args.e2e_steps)}))
        return
    savers = load_savers()
    out = {'card': card(), 'cpu_threads': torch.get_num_threads(),
           'per_frame_1080p': per_frame(savers, args.frames, args.ref_frames), 'pil_encode_1080p_ms': encode_ms(),
           'e2e_demo_1080p_in_480p_work': e2e(savers, args.e2e_steps, args.ref_e2e_steps)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
