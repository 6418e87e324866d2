"""Frames per second of the demos' loop (demo/demo_automatic.py) with three ingests.

    python tools/bench_demo.py [--frames 60] [--size 480] [--out results/bench_demo.json]

A seeded 1080p q90 JPEG folder is read by ``SimpleVideoReader`` and run through the reference's unmodified
``process_frame_automatic`` and ``flush_buffer`` (staged under oracle/_ref by oracle/build_ref_demo.py), the DEVA network
with a synthetic checkpoint, and this package's ``ResultSaver`` in demo mode with the device PNG and JPEG encoders.
SAM is the detector fake of tests/golden/detector_masks_scenario.py: it returns five seeded masks at once, so the
detector network's time is excluded (in the real semionline demo SAM runs on 3 frames in 5 and dominates wall time).
Modes: online (``detection_every`` 5) and semionline (the defaults).  Arms:
  * ``reference_ingest``: ``DataLoader(reader, batch_size=None, collate_fn=no_collate, num_workers=8)`` and the
    reference's own ``demo_utils.get_input_frame_for_deva`` (host float32 normalise and ``F.interpolate``, then
    ``.cuda()``), set on the loaded processor module, which binds it at import;
  * ``dataloader``: the same DataLoader with this package's ``get_input_frame_for_deva`` (the gradio demo's numpy path);
  * ``device_loader``: ``DeviceLoader(reader)``, CUDA frames throughout.
Ingest time per frame is the host time spent waiting for the loader's next frame plus the time in
``get_input_frame_for_deva``.  One JSON line, with the card, its power limit and the host's CPU count read in the same
run.
"""
import argparse
import json
import os
import sys
import tempfile
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, 'oracle', '_ref')
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (puts the package on sys.path)

sys.path.append(REF)  # after the package: the staged processors and the reference's deva.dataset
sys.path.append(GOLDEN)
import importlib.util  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402
from torch.utils.data import DataLoader  # noqa: E402

import demo_scenario as sc  # noqa: E402
import detector_masks_scenario as dms  # noqa: E402
from bench_reader import card  # noqa: E402

H, W = 1080, 1920
CFG = dict(key_dim=64, value_dim=512, pix_feat_dim=512, mem_every=5, enable_long_term=True, chunk_size=-1, top_k=30,
           enable_long_term_count_usage=False, max_mid_term_frames=10, min_mid_term_frames=5, num_prototypes=128,
           max_long_term_elements=10000)


def make_folder(root, frames):
    os.makedirs(root)
    rng = np.random.default_rng(0)
    base = np.asarray(Image.fromarray(rng.integers(0, 256, (H // 16 + 1, W // 16 + 1, 3), dtype=np.uint8)).resize(
        (W, H), Image.BILINEAR))
    for t in range(frames):
        Image.fromarray(np.roll(base, 4 * t, axis=1)).save(os.path.join(root, f'{t:05d}.jpg'), quality=90)
    return root


def load_reference_demo_utils():
    spec = importlib.util.spec_from_file_location('ref_demo_utils', os.path.join(REF, 'deva', 'inference',
                                                                                 'demo_utils.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class Timed:
    """Iterates ``loader``, adding the host time spent waiting for each item to ``clock``."""

    def __init__(self, loader, clock):
        self.loader, self.clock = loader, clock

    def __iter__(self):
        it = iter(self.loader)
        while True:
            t0 = time.perf_counter()
            try:
                item = next(it)
            except StopIteration:
                return
            self.clock[0] += time.perf_counter() - t0
            yield item


def run(processors, ingest, loader, temporal, size, sd, masks, out):
    """One demo loop; -> (seconds to the saver's end and a device synchronise, ingest seconds)."""
    from deva.inference.demo_utils import flush_buffer
    from deva.inference.inference_core import DEVAInferenceCore
    from deva.inference.result_utils import ResultSaver
    from deva.model.network import DEVA
    clock = [0.0]

    def timed_ingest(image_np, min_side):
        t0 = time.perf_counter()
        x = ingest(image_np, min_side)
        clock[0] += time.perf_counter() - t0
        return x
    processors.get_input_frame_for_deva = timed_ingest
    np.random.seed(42)
    cfg = dict(sc.demo_config(CFG, 'auto', temporal), size=size)
    net = DEVA(cfg).cuda().eval()
    net.load_weights(sd)
    deva = DEVAInferenceCore(net, config=cfg)
    saver = ResultSaver(out, None, dataset='demo', object_manager=deva.object_manager, png_encoder='device',
                        jpeg_encoder='device')
    sam = dms.FakeAutoSam(masks, dms.iou_preds(len(masks), 1), 'cuda')
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.inference_mode():
        sc.run_demo(processors, flush_buffer, deva, Timed(loader, clock), 'auto', saver, (sam, ))
    saver.end()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, clock[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=60)
    ap.add_argument('--size', type=int, default=480)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from deva import _native
    from deva.inference import demo_utils
    from deva.inference.data.device_loader import DeviceLoader
    from deva.inference.data.simple_video_reader import SimpleVideoReader, no_collate
    from deva.model.param_spec import synthetic_state_dict
    _native.require_device()
    torch.cuda.set_device(0)
    torch.autograd.set_grad_enabled(False)
    dms.install_detector_stubs([])
    from deva.ext import automatic_processor
    if not automatic_processor.__file__.startswith(REF):
        raise RuntimeError('the demo processors are not staged: run python oracle/build_ref_demo.py in the build '
                           'container')
    ref = load_reference_demo_utils()
    sd = {k: v.cuda() for k, v in synthetic_state_dict(seed=1).items()}
    masks = dms.build_masks([('rand', 5)], H, W, 1)
    result = {'card': card(), 'host_cpus': os.cpu_count(), 'frames': args.frames, 'size': args.size,
              'source': f'{W}x{H} q90 JPEG', 'detector': 'fake SAM (seeded masks, no network): detector time excluded',
              'saver': 'demo, device PNG and JPEG encoders', 'modes': {}}
    with tempfile.TemporaryDirectory() as tmp:
        folder = make_folder(os.path.join(tmp, 'frames'), args.frames)

        def dataloader():
            return DataLoader(SimpleVideoReader(folder), batch_size=None, collate_fn=no_collate, num_workers=8)
        arms = {'reference_ingest': (ref.get_input_frame_for_deva, dataloader),
                'dataloader': (demo_utils.get_input_frame_for_deva, dataloader),
                'device_loader': (demo_utils.get_input_frame_for_deva, lambda: DeviceLoader(SimpleVideoReader(folder)))}
        for temporal in ('online', 'semionline'):
            res = {}
            for rep in range(2):  # the first pass warms every shape up; the second is reported
                for name, (ingest, loader) in arms.items():
                    secs, ingest_secs = run(automatic_processor, ingest, loader(), temporal, args.size, sd, masks,
                                            os.path.join(tmp, f'{temporal}_{name}_{rep}'))
                    if rep:
                        res[name] = {'fps': round(args.frames / secs, 2),
                                     'ingest_ms_per_frame': round(1e3 * ingest_secs / args.frames, 2)}
            result['modes'][temporal] = res
            print(temporal, res, flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or '.', exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
