"""Images of the PNG encoder tests (tests/test_png_encode_cpu.py against Pillow, tests/test_png_encode_gpu.py against
oracle/png_encode.py), regenerated from their case ids: '<mode>-<content>-<h>x<w>'.

mode: L, RGB or P<n> (a P image whose palette has n colours); content: 'const' (one value beyond small palettes),
'ellipse' (a segmentation map of 16 overlapping ellipses), 'noise' (uniform bytes) or 'run' (constant rows whose first
pixel differs, so every row segment ends in a run of w - 2 equal bytes: 254 to 259 for the widths below)."""
import numpy as np

MODES = ['L', 'RGB', 'P2', 'P4', 'P16', 'P17', 'P256']
SMALL_SHAPES = [(1, 1), (1, 37), (29, 1), (13, 7), (9, 13), (37, 53)]
RUN_WIDTHS = [256, 257, 258, 259, 260, 261]
LAYOUTS = [('L', None), ('RGB', None)] + [('P', [(7 * i) % 256 for i in range(3 * n)]) for n in (1, 2, 3, 4, 5, 16, 17,
                                                                                                    255, 256)] + \
    [('P', None), ('P', bytes(range(256)) * 3)]


def case_ids(large):
    if not large:
        ids = [f'{m}-{c}-{h}x{w}' for m in MODES for c in ('const', 'ellipse', 'noise') for h, w in SMALL_SHAPES]
        return ids + [f'{m}-run-3x{w}' for m in ('L', 'RGB', 'P4') for w in RUN_WIDTHS]
    ids = [f'{m}-ellipse-1080x1920' for m in MODES] + [f'{m}-const-1080x1920' for m in ('L', 'RGB', 'P2')]
    ids += [f'{m}-ellipse-2160x3840' for m in ('L', 'RGB', 'P16', 'P256')]
    return ids + [f'{m}-noise-1080x1920' for m in ('L', 'RGB', 'P4')]


def palette(n):
    return [(37 * i + 11) % 256 for i in range(3 * n)]


def ellipses(h, w, k=16, seed=0):
    rng = np.random.default_rng(seed)
    ids = np.zeros((h, w), np.int32)
    yy, xx = np.ogrid[:h, :w]
    for i in range(1, k + 1):
        cy, cx = rng.uniform(0, h), rng.uniform(0, w)
        ry, rx = rng.uniform(h / 20, h / 4) + 0.5, rng.uniform(w / 20, w / 4) + 0.5
        ids[((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1] = i
    return ids


def make(case):
    """-> (uint8 image, PIL mode, palette or None)."""
    mode, content, shape = case.split('-')
    h, w = (int(v) for v in shape.split('x'))
    rng = np.random.default_rng([ord(c) for c in case])
    if content == 'const':
        ids = np.full((h, w), 200, np.int32)
    elif content == 'ellipse':
        ids = ellipses(h, w) * 37 % 256
    elif content == 'noise':
        ids = rng.integers(0, 256, (h, w))
    else:
        ids = np.full((h, w), 9, np.int32)
        ids[:, 0] = np.arange(h) + 1
    if mode == 'RGB':
        if content == 'noise':
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        else:
            lut = rng.integers(0, 256, (256, 3), dtype=np.uint8)
            img = lut[ids]
        return np.ascontiguousarray(img), 'RGB', None
    img = ids.astype(np.uint8)
    if mode == 'L':
        return img, 'L', None
    return img, 'P', palette(int(mode[1:]))
