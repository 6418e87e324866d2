"""Time SAM's automatic mask generation per frame: the reference SamAutomaticMaskGenerator (staged unmodified under
oracle/_ref by oracle/build_ref_sam.py) against deva.ext.sam_masks.DeviceMaskGenerator, on the same GPU, over
oracle/sam_stub.py's FakeSam (no image encoder; its mask decoder runs in both legs and is timed on its own).

    python tools/bench_sam_masks.py [--reps 5] [--out FILE]

At 1080p with 32 and 64 points per side, from scratch and with a semionline positive-point subset, prints one JSON line:
reference and device ms per generate call, the time of set_image and the fake decoder alone (in both), the peak device
memory each call adds, the device kernels' time from CUDA events (statistics over one batch, and the mask writer over the kept masks), whether every field is equal, and the
card's name, power limit and SM clock.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tracking-anything-with-deva_b200'), os.path.join(ROOT, 'tests', 'golden')]

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = 'name,power.limit,clocks.max.sm,clocks.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True,
                             text=True, check=True).stdout.strip().splitlines()[0]
        return dict(zip(q.split(','), [s.strip() for s in out.split(',')]))
    except Exception as e:  # reported, not fatal: the timings stand on their own
        return {'error': str(e)}


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    times, peaks = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t) * 1e3)
        peaks.append(torch.cuda.max_memory_allocated() - base)
        del out
    return float(np.median(times)), float(min(times)), int(max(peaks))


def same(a, b):
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.is_floating_point():
        a, b = a.cpu(), b.cpu()
        return torch.equal(a.isnan(), b.isnan()) and torch.equal(a[~a.isnan()], b[~b.isnan()])
    return torch.equal(a.cpu(), b.cpu())


def decoder_ms(gen, img, pos, reps=3):
    """Host-clock time of set_image plus the fake decoder over every batch: the part both legs share."""
    h, w = img.shape[:2]
    pts = (pos if pos is not None else gen.point_grid) * np.array([[w, h]])

    def run():
        gen.predictor.set_image(img)
        for b in range(0, len(pts), gen.points_per_batch):
            gen._decode(pts[b:b + gen.points_per_batch], None, (h, w))
        gen.predictor.reset_image()
    return timed(run, reps)[0]


def kernel_ms(nat, gen, img, reps=20):
    """CUDA-event time of the statistics kernel over one batch of 3 x points_per_batch candidates and of the mask
    writer over the masks the frame keeps."""
    h, w = img.shape[:2]
    pred = gen.predictor
    pred.set_image(img)
    in_h, in_w = pred.input_size
    _, low_res, iou = gen._decode(gen.point_grid[:gen.points_per_batch] * np.array([[w, h]]), None, (h, w))
    logits, iou = low_res.flatten(0, 1).contiguous(), iou.flatten(0, 1).contiguous()
    stats = torch.empty(logits.shape[0], nat.SAM_STATS, dtype=torch.int32, device='cuda')
    out = gen.generate(img)
    k = out['masks'].shape[0]
    sel = torch.arange(k, device='cuda') % logits.shape[0]
    masks = torch.empty(k, h, w, dtype=torch.bool, device='cuda')
    res = {}
    for name, fn in (('stats_batch', lambda: nat.sam_mask_stats(logits, 1024, in_h, in_w, h, w, iou, 0.88, 1.0, -1.0,
                                                                 0.0, stats)),
                     ('stats_batch_all', lambda: nat.sam_mask_stats(logits, 1024, in_h, in_w, h, w, None, 0.0, 1.0,
                                                                     -1.0, 0.0, stats)),
                     ('write_kept', lambda: nat.sam_mask_write(logits, sel, 1024, in_h, in_w, h, w, 0.0, masks))):
        fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        res[name + '_ms'] = round(a.elapsed_time(b) / reps, 4)
    res['batch_candidates'] = int(logits.shape[0])
    res['batch_candidates_above_iou'] = int((iou > 0.88).sum())
    res['kept_masks'] = k
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from deva import _native as nat
    nat.require_device()
    from oracle import sam_masks, sam_stub
    RefGen = sam_masks.reference_generator()
    from deva.ext.sam_masks import DeviceMaskGenerator
    import sam_masks_scenario as sc
    h, w = 1080, 1920
    img = sc.image(h, w, 0)
    rows = []
    for pps in (32, 64):
        for subset in (False, True):
            model = sam_stub.FakeSam(seed=pps).cuda()
            pos = sc._subset(pps, 0.25, 1) if subset else None
            ref = RefGen(model, points_per_side=pps, points_per_batch=64, pred_iou_thresh=0.88)
            dev = DeviceMaskGenerator(model, points_per_side=pps, points_per_batch=64, pred_iou_thresh=0.88)
            a, b = ref.generate(img, pos), dev.generate(img, pos)
            equal = {k: same(a[k], b[k]) for k in ('masks', 'iou_preds', 'points', 'stability_score', 'boxes')}
            del a, b
            r_med, r_min, r_peak = timed(lambda: ref.generate(img, pos), args.reps)
            d_med, d_min, d_peak = timed(lambda: dev.generate(img, pos), args.reps)
            row = dict(points_per_side=pps, prompts=len(pos) if subset else pps * pps, subset=subset,
                       reference_ms=round(r_med, 2), reference_min_ms=round(r_min, 2),
                       reference_peak_extra_mib=round(r_peak / 2 ** 20, 1), device_ms=round(d_med, 2),
                       device_min_ms=round(d_min, 2), device_peak_extra_mib=round(d_peak / 2 ** 20, 1),
                       speedup=round(r_med / d_med, 2), candidates_before_nms=dev.candidates, equal=equal)
            row['decoder_ms'] = round(decoder_ms(dev, img, pos), 2)
            row.update(kernel_ms(nat, dev, img))
            rows.append(row)
            print(json.dumps(row), file=sys.stderr)
    result = {'frame': [h, w], 'model': 'oracle.sam_stub.FakeSam', 'reps': args.reps, 'card': card(), 'rows': rows,
              'all_equal': all(all(r['equal'].values()) for r in rows)}
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, 'w').write(line + '\n')


if __name__ == '__main__':
    main()
