"""Detector masks -> detection id map (``auto_segment``, ``segment_with_text``) - the reference's and this package's.

    python tools/bench_detector_masks.py [--reps 10] [--ref-reps 3]

Input: a seeded 1080p frame, working resolution min_side = 480 (480x853), with detector fakes (the fixture's, from
tests/golden/detector_masks_scenario.py) in place of SAM and Grounding-DINO:
  * automatic: SAM's generator returns N in {32, 128, 256} random blob masks, bool, already on the device (as DEVA's
    generator returns them), suppress_small_mask on and off;
  * text: N in {5, 20, 50} boxes; the predictor returns three nested box masks per box on the host, as SamPredictor does.
Reference: the unmodified ``deva/ext/automatic_sam.py`` / ``grounding_dino.py`` staged under oracle/_ref by
oracle/build_ref_ext.py, loaded by path with stub detector modules.  Ours: ``deva.ext.automatic_sam`` /
``deva.ext.grounding_dino``.  Per workload:
  * ms per call: host clock around calls that end in their own synchronisation;
  * the kernels alone (CUDA events over repeated launches, masks resident) and the mask bytes they read (each kernel
    pass reads every mask once) over that time, as a share of the H100 SXM's 3.35 TB/s;
  * peak extra device memory of one call (max_memory_allocated over what was allocated before it);
  * whether the two id maps are equal.
Prints one JSON line with the card and its power limit read in the same run."""
import argparse
import importlib.util
import json
import os
import sys
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, 'oracle', '_ref', 'deva', 'ext')
sys.path.insert(0, ROOT)
import bench  # noqa: E402,F401  (puts the package on sys.path)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import detector_masks_scenario as sc  # noqa: E402
from bench_ingest import card  # noqa: E402

H, W, MIN_SIDE = 1080, 1920, 480
HBM_TBPS = 3.35


def load_reference(name):
    file = os.path.join(REF, f'{name}.py')
    if not os.path.isfile(file):
        raise RuntimeError('oracle/_ref/deva/ext is not staged: run python oracle/build_ref_ext.py in the build container')
    spec = importlib.util.spec_from_file_location(f'ref_{name}', file)  # not deva.ext.*: those are ours
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def blob_masks(n, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    coarse = torch.rand((n, 1, H // 64, W // 64), generator=g, device='cuda')
    blobs = F.interpolate(coarse, (H, W), mode='bilinear', align_corners=False)[:, 0]
    return (blobs > torch.rand((n, 1, 1), generator=g, device='cuda') * 0.5 + 0.45).contiguous()


def text_boxes(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        x0, y0 = int(rng.integers(0, W - 400)), int(rng.integers(0, H - 300))
        out.append((x0, y0, x0 + int(rng.integers(20, 400)), y0 + int(rng.integers(20, 300)), 0.9 - i * 0.01, i % 4))
    return out


def per_call(fn, reps):
    """-> (ms per call, peak extra device MB of one call, last result)."""
    out = fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps, peak, out


def event_ms(fn, reps):
    fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def kernel_figures(ms, mask_bytes):
    rate = mask_bytes / (ms * 1e-3) / 1e12
    return {'kernels_ms': round(ms, 4), 'mask_bytes_read_MB': round(mask_bytes / 1e6, 1),
            'TBps': round(rate, 3), 'share_of_3.35TBps': round(rate / HBM_TBPS, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--ref-reps', type=int, default=3)
    args = ap.parse_args()
    from deva import _native as nat
    nat.require_device()
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    sc.install_detector_stubs([])
    sc.checksum = lambda a: 0  # the fakes' call records checksum every image: test bookkeeping, not detector work
    ref_auto, ref_text = load_reference('automatic_sam'), load_reference('grounding_dino')
    from deva.ext.automatic_sam import auto_segment
    from deva.ext.grounding_dino import segment_with_text
    img = sc.image(H, W)
    oh, ow = int(H * MIN_SIDE / H), int(W * MIN_SIDE / H)
    rows = []
    for n in (32, 128, 256):
        masks = blob_masks(n, n)
        iou = torch.rand(n, device='cuda')
        sam = sc.FakeAutoSam(np.zeros((0, 1, 1), bool), np.zeros(0, np.float32), 'cuda')
        sam.masks, sam.iou_preds = masks, iou
        for suppress in (True, False):
            cfg = sc.auto_config(0.8)
            ours_ms, ours_mb, (ours_map, ours_seg) = per_call(
                lambda: auto_segment(cfg, sam, img, None, MIN_SIDE, suppress), args.reps)
            ref_ms, ref_mb, (ref_map, ref_seg) = per_call(
                lambda: ref_auto.auto_segment(cfg, sam, img, None, MIN_SIDE, suppress), args.ref_reps)
            area = torch.empty(n, device='cuda')
            slot = torch.empty((oh, ow), dtype=torch.int32, device='cuda')
            won = torch.empty(n + 1, dtype=torch.int32, device='cuda')
            kept = torch.empty_like(won)

            def kernels():
                nat.mask_stats(masks, oh, ow, area, None)
                nat.mask_scored_argmax(masks, oh, ow, area, suppress, slot, won, kept)
            rows.append(dict({'path': 'auto', 'n': n, 'suppress_small_mask': suppress,
                              'ours_ms': round(ours_ms, 3), 'reference_ms': round(ref_ms, 3),
                              'speedup': round(ref_ms / ours_ms, 1), 'ours_peak_extra_MB': round(ours_mb, 1),
                              'reference_peak_extra_MB': round(ref_mb, 1),
                              'maps_equal': bool(torch.equal(ours_map, ref_map)),
                              'segments_equal': [(s.id, s.scores) for s in ours_seg] ==
                                                [(s.id, s.scores) for s in ref_seg]},
                             **kernel_figures(event_ms(kernels, args.reps), 2 * n * H * W)))
    for n in (5, 20, 50):
        boxes = text_boxes(n, n)
        cfg = sc.text_config(0.8)
        ours_ms, ours_mb, (ours_map, ours_seg) = per_call(
            lambda: segment_with_text(cfg, sc.FakeGroundingDino(boxes, 'cuda'), sc.FakeSamPredictor(), img, ['a'],
                                      MIN_SIDE), args.reps)
        ref_ms, ref_mb, (ref_map, ref_seg) = per_call(
            lambda: ref_text.segment_with_text(cfg, sc.FakeGroundingDino(boxes, 'cuda'), sc.FakeSamPredictor(), img,
                                               ['a'], MIN_SIDE), args.ref_reps)
        # the kernel alone, on the same mask stack uploaded once
        sam = sc.FakeSamPredictor()
        sam.set_image(img)
        stack = torch.from_numpy(np.stack([sam.predict(np.array(b[:4], np.float32), True)[0][0] for b in boxes])).cuda()
        order = torch.arange(n, dtype=torch.int32, device='cuda')
        slot = torch.empty((oh, ow), dtype=torch.int32, device='cuda')
        covered = torch.empty(n, dtype=torch.int32, device='cuda')
        ms = event_ms(lambda: nat.mask_last_cover(stack, oh, ow, order, slot, covered), args.reps)
        rows.append(dict({'path': 'text', 'n': n, 'ours_ms': round(ours_ms, 3), 'reference_ms': round(ref_ms, 3),
                          'speedup': round(ref_ms / ours_ms, 1), 'ours_peak_extra_MB': round(ours_mb, 1),
                          'reference_peak_extra_MB': round(ref_mb, 1),
                          'maps_equal': bool(torch.equal(ours_map, ref_map)),
                          'segments_equal': [(s.id, s.scores) for s in ours_seg] == [(s.id, s.scores) for s in ref_seg]},
                         **kernel_figures(ms, n * H * W)))
    print(json.dumps({'card': card(), 'frame': [H, W], 'min_side': MIN_SIDE, 'out': [oh, ow], 'reps': args.reps,
                      'ref_reps': args.ref_reps, 'rows': rows}))


if __name__ == '__main__':
    main()
