"""numpy restatement of the detector-mask compositions (deva/ext/detector_masks.py) - test oracle only.

``resize`` is the bilinear arithmetic the kernels compile to for mask bytes (align_corners=False, the same-size copy):
the source index fma(scale, dst + 0.5, -0.5) and the row blend fma(ly0, top, ly1 * bot), fused multiply-adds emulated
in float64 (exact product, then rounding).  That is also what torch's CPU kernel computes: the plain float32 formula, one
rounding per operation, differs from it in the last bits, and at scales where a value lands next to 0.5 it makes
different > 0.5 decisions.  The rules are the reference's: auto_segment's scored argmax with its acceptance rule in
float32, and segment_with_text's paint order by descending int64 pixel count.
"""
import numpy as np


def _fma(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def _taps(n_in, n_out):
    r = np.float32(n_in / n_out)
    s = np.maximum(_fma(r, np.arange(n_out, dtype=np.float32) + np.float32(0.5), -0.5), np.float32(0))
    i0 = s.astype(np.int64)
    l1 = (s - i0.astype(np.float32)).astype(np.float32)
    return i0, np.minimum(i0 + 1, n_in - 1), (np.float32(1) - l1).astype(np.float32), l1


def resize(masks: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """[n, h, w] bool / uint8 (0 / 1) -> float32 [n, out_h, out_w].  With 0 / 1 taps the column blends are exact sums of
    weights, so only the row blend's fusing matters."""
    m = masks.astype(np.float32)
    if m.shape[1:] == (out_h, out_w):
        return m
    y0, y1, ly0, ly1 = _taps(m.shape[1], out_h)
    x0, x1, lx0, lx1 = _taps(m.shape[2], out_w)
    top = (lx0 * m[:, y0][:, :, x0] + lx1 * m[:, y0][:, :, x1]).astype(np.float32)
    bot = (lx0 * m[:, y1][:, :, x0] + lx1 * m[:, y1][:, :, x1]).astype(np.float32)
    return _fma(ly0[:, None], top, (ly1[:, None] * bot).astype(np.float32))


def scored_id_map(masks, iou_preds, out_h, out_w, suppress_small_mask, overlap_threshold):
    """-> (int64 [out_h, out_w], [(id, score)]): auto_segment's map and segments."""
    n = masks.shape[0]
    if n == 0:
        return np.zeros((out_h, out_w), np.int64), []
    v = resize(masks, out_h, out_w)
    area = v.reshape(n, -1).sum(1, dtype=np.float32)
    score = area if suppress_small_mask else (area.max() * np.float32(2) - area).astype(np.float32)
    scored = np.concatenate([np.full((1, out_h, out_w), 0.1, np.float32), v * score[:, None, None]])
    hard = scored.argmax(0)
    segments = []
    if not suppress_small_mask:
        for k in range(n):
            if (hard == k + 1).any():
                segments.append((len(segments) + 1, float(iou_preds[k])))
        return hard.astype(np.int64), segments
    out = np.zeros((out_h, out_w), np.int64)
    for k in range(n):
        won, covered = int((hard == k + 1).sum()), int((v[k] > 0.5).sum())
        paint = (hard == k + 1) & (v[k] >= 0.5)
        if won > 0 and covered > 0 and paint.any():
            if np.float32(won) / np.float32(covered) < np.float32(overlap_threshold):
                continue
            segments.append((len(segments) + 1, float(iou_preds[k])))
            out[paint] = len(segments)
    return out, segments


def cover_id_map(masks, out_h, out_w):
    """-> (int64 [out_h, out_w], [(id, mask index)]): segment_with_text's map, painting in descending pixel count."""
    out = np.zeros((out_h, out_w), np.int64)
    segments = []
    if len(masks) == 0:
        return out, segments
    v = resize(np.asarray(masks), out_h, out_w)
    areas = np.array([np.count_nonzero(m) for m in masks], dtype=np.int64)
    for i in np.flip(np.argsort(areas)):
        on = v[i] > 0.5
        if on.any():
            segments.append((len(segments) + 1, int(i)))
            out[on] = len(segments)
    return out, segments
