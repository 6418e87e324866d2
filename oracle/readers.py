"""Host oracle of the dataset readers' mask transforms, restated in numpy from libImaging and the readers' arithmetic.

* ``pil_bilinear_coeffs`` / ``pil_resample``: Pillow's ``Image.resize(size, BILINEAR)`` of an 8-bit one-channel image
  (Resample.c: precompute_coeffs with the triangle filter, normalize_coeffs_8bpc to 22-bit fixed point, the horizontal
  pass, clip8, then the vertical pass; a pass whose axis keeps its size is skipped).  Written per output pixel with
  Python scalars, the way the C loops read, so it shares no code with the package's vectorised tables.
* ``rgb_ids_nearest``: the detection reader's ``Resize(NEAREST)`` of an RGB mask and its ``r + 256 g + 65536 b`` id
  map, from PIL's nearest source index along each axis.
"""
import math

import numpy as np

PRECISION_BITS = 22


def pil_bilinear_coeffs(n_in: int, n_out: int):
    """[(first input index, [fixed-point coefficient per tap])] per output pixel."""
    scale = float(np.float32(n_in)) / n_out
    filterscale = scale if scale >= 1.0 else 1.0
    support = 1.0 * filterscale
    out = []
    for xx in range(n_out):
        center = (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), n_in) - xmin
        ws, ww = [], 0.0
        for x in range(xmax):
            t = abs((x + xmin - center + 0.5) * ss)
            wt = 1.0 - t if t < 1.0 else 0.0
            ws.append(wt)
            ww += wt
        if ww != 0.0:
            ws = [wt / ww for wt in ws]
        out.append((xmin, [int(-0.5 + wt * (1 << PRECISION_BITS)) if wt < 0 else int(0.5 + wt * (1 << PRECISION_BITS))
                           for wt in ws]))
    return out


def _pass(img: np.ndarray, coeffs) -> np.ndarray:
    """One pass along the last axis of int64 ``img``."""
    out = np.empty(img.shape[:-1] + (len(coeffs),), np.int64)
    for o, (lo, ks) in enumerate(coeffs):
        ss = np.full(img.shape[:-1], 1 << (PRECISION_BITS - 1), np.int64)
        for j, k in enumerate(ks):
            ss += img[..., lo + j] * k
        out[..., o] = np.clip(ss >> PRECISION_BITS, 0, 255)
    return out


def pil_resample(img: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """uint8 [h, w] -> uint8 [out_h, out_w]: ``np.asarray(Image.fromarray(img).resize((out_w, out_h), BILINEAR))``."""
    h, w = img.shape
    x = img.astype(np.int64)
    if out_w != w:
        x = _pass(x, pil_bilinear_coeffs(w, out_w))
    if out_h != h:
        x = _pass(x.T, pil_bilinear_coeffs(h, out_h)).T
    return x.astype(np.uint8)


def nearest_map(n_in: int, n_out: int) -> np.ndarray:
    """PIL's NEAREST source index along one axis: a double coordinate from 0.5 * n_in / n_out stepped by n_in / n_out,
    truncated (ImagingScaleAffine)."""
    a = n_in / n_out
    xo, out = a * 0.5, []
    for _ in range(n_out):
        out.append(min(math.floor(xo), n_in - 1))
        xo += a
    return np.array(out, np.int64)


def rgb_ids_nearest(rgb: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """uint8 [h, w, 3] -> int32 [out_h, out_w]: the nearest resize, then r + 256 g + 65536 b."""
    h, w, _ = rgb.shape
    m = rgb[nearest_map(h, out_h)][:, nearest_map(w, out_w)].astype(np.int32)
    return m[..., 0] + m[..., 1] * 256 + m[..., 2] * 65536
