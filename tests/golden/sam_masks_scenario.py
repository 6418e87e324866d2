"""Scenarios of tests/golden/sam_masks.{json,npz}: SAM's automatic mask generator over oracle/sam_stub.py's FakeSam.

Each case is one ``generate`` call: frame size, FakeSam knobs, generator arguments and prompts.  They cover 32 and 64
points per side with points_per_batch not dividing the prompt count, positive-point subsets (the semionline forward
mask's background points, an empty set included) and negative points, landscape / portrait / odd / smaller-than-1024
frames and a 1080p one, batches filtered whole by predicted IoU, a frame with no masks, masks entirely below -1 (zero
unions), masks touching the border, and predicted IoUs on a 1/32 grid, so NMS sees ties."""
import numpy as np

from oracle.sam_stub import build_point_grid


def _subset(n_per_side, keep_fraction, seed):
    """Grid points outside a seeded disc: the points a forward mask leaves as background."""
    pts = build_point_grid(n_per_side).astype(np.float32)
    rng = np.random.default_rng(seed)
    c, r = rng.uniform(0.3, 0.7, 2), np.sqrt(1 - keep_fraction) * 0.6
    return pts[np.hypot(pts[:, 0] - c[0], pts[:, 1] - c[1]) > r]


def image(h, w, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


CASES = {
    'grid32_landscape': dict(h=480, w=640, seed=0, pps=32, ppb=100),
    'grid64_portrait_small': dict(h=300, w=200, seed=1, pps=64, ppb=500),
    'grid16_odd_subset_negative': dict(h=333, w=517, seed=2, pps=16, ppb=64, positive=(16, 0.6, 2),
                                       negative=[[0.2, 0.3], [0.7, 0.6]]),
    'grid32_filtered_batches': dict(h=720, w=1280, seed=3, pps=32, ppb=64, low_iou_top=0.35),
    'grid32_dead_masks': dict(h=512, w=512, seed=4, pps=32, ppb=48, dead=0.5),
    'grid16_no_masks': dict(h=240, w=320, seed=5, pps=16, ppb=64, low_iou_top=1.1),
    'grid16_thresholds': dict(h=400, w=300, seed=6, pps=16, ppb=30, pred_iou=0.0, stability=0.0, offset=0.5,
                              nms=0.5),
    'grid32_1080p_subset': dict(h=1080, w=1920, seed=7, pps=32, ppb=64, positive=(32, 0.12, 7)),
    'grid32_empty_subset': dict(h=240, w=320, seed=8, pps=32, ppb=64, positive_empty=True),
}


def arguments(case):
    """-> (FakeSam kwargs, generator kwargs, image, positive_points, negative_points)"""
    c = CASES[case]
    model = dict(seed=c['seed'], low_iou_top=c.get('low_iou_top', 0.0), dead=c.get('dead', 0.04))
    gen = dict(points_per_side=c['pps'], points_per_batch=c['ppb'], pred_iou_thresh=c.get('pred_iou', 0.88),
               stability_score_thresh=c.get('stability', 0.95), stability_score_offset=c.get('offset', 1.0),
               box_nms_thresh=c.get('nms', 0.7))
    pos = _subset(*c['positive']) if 'positive' in c else None
    if c.get('positive_empty'):
        pos = np.zeros((0, 2), dtype=np.float32)
    neg = np.array(c['negative'], dtype=np.float32) if 'negative' in c else None
    return model, gen, image(c['h'], c['w'], c['seed']), pos, neg
