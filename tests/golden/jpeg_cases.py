"""Images of the JPEG encoder tests (tests/test_jpeg_encode_cpu.py against Pillow, tests/test_jpeg_encode_gpu.py against
oracle/jpeg_encode.py), regenerated from their case ids: '<content>-<h>x<w>-q<quality>'.

content: 'const' (one colour), 'gradient' (smooth ramps), 'noise' (uniform bytes), 'saturated' (every channel 0 or
255), 'overlay' (a demo overlay: a smooth frame blended half and half with the colours of 16 overlapping ellipses, so
flat regions and hard edges) or 'rand<seed>' (uniform bytes from numpy's PCG64 at that seed: the fill cases below end
their scan in a 0xFF byte made by the 1-bit fill, which is then stuffed)."""
import numpy as np

SHAPES = [(1, 1), (1, 17), (7, 9), (8, 8), (15, 17), (16, 16), (17, 31), (33, 17), (37, 53), (120, 200), (481, 857)]
CONTENTS = ['const', 'gradient', 'noise', 'saturated', 'overlay']
QUALITIES = [1, 10, 50, 90, 95, 100]
# every h mod 16 and every w mod 16 ((5 r + 3) mod 16 runs through all residues)
RESIDUES = [(32 + r, 48 + (5 * r + 3) % 16) for r in range(16)]
FILL_FF = ['rand13-8x8-q100', 'rand27-8x8-q95']


def case_ids(large):
    if large:
        return [f'{c}-1080x1920-q75' for c in ('overlay', 'noise')]
    ids = [f'{c}-{h}x{w}-q75' for c in CONTENTS for h, w in SHAPES]
    ids += [f'{c}-{h}x{w}-q75' for c in ('overlay', 'noise') for h, w in RESIDUES]
    ids += [f'{c}-{h}x{w}-q{q}' for q in QUALITIES for c in ('overlay', 'noise', 'gradient') for h, w in [(37, 53)]]
    ids += [f'noise-120x200-q{q}' for q in QUALITIES]
    return ids + FILL_FF


def ellipses(h, w, k=16, seed=0):
    rng = np.random.default_rng(seed)
    ids = np.zeros((h, w), np.int32)
    yy, xx = np.ogrid[:h, :w]
    for i in range(1, k + 1):
        cy, cx = rng.uniform(0, h), rng.uniform(0, w)
        ry, rx = rng.uniform(h / 20, h / 4) + 0.5, rng.uniform(w / 20, w / 4) + 0.5
        ids[((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1] = i
    return ids


def frame(h, w, seed=0):
    """A smooth, natural-looking uint8 RGB frame: low-frequency colour waves with a little grain."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:h, :w].astype(np.float32)
    out = np.empty((h, w, 3), np.float32)
    for c in range(3):
        fy, fx, ph = rng.uniform(1, 4) / max(h, 1), rng.uniform(1, 4) / max(w, 1), rng.uniform(0, 6.3)
        out[..., c] = 128 + 90 * np.sin(2 * np.pi * (fy * yy + fx * xx) + ph)
    out += rng.normal(0, 4, out.shape)
    return np.clip(out, 0, 255).astype(np.uint8)


def overlay(h, w, k=16, seed=0):
    """The saver's demo blend of ``frame`` with the colours of ``k`` ellipse ids: alpha 1 where the id is 0, else 0.5."""
    ids = ellipses(h, w, k, seed)
    colours = np.random.default_rng(seed + 1).integers(0, 256, (k + 1, 3)).astype(np.float32)
    alpha = (ids == 0).astype(np.float32)[:, :, None] * 0.5 + 0.5
    return (frame(h, w, seed) * alpha + colours[ids] * (1 - alpha)).astype(np.uint8)


def make(case):
    """-> (uint8 RGB image [h, w, 3], quality)."""
    content, shape, q = case.split('-')
    h, w = (int(v) for v in shape.split('x'))
    rng = np.random.default_rng([ord(c) for c in case])
    if content == 'const':
        img = np.broadcast_to(rng.integers(0, 256, 3, dtype=np.uint8), (h, w, 3))
    elif content == 'gradient':
        yy, xx = np.mgrid[:h, :w]
        img = np.stack([(yy * 255) // max(h - 1, 1), (xx * 255) // max(w - 1, 1), ((yy + xx) * 3) % 256], -1)
    elif content == 'noise':
        img = rng.integers(0, 256, (h, w, 3))
    elif content == 'saturated':
        img = rng.integers(0, 2, (h, w, 3)) * 255
    elif content == 'overlay':
        img = overlay(h, w)
    else:
        assert content.startswith('rand'), case
        img = np.random.default_rng(int(content[4:])).integers(0, 256, (h, w, 3), dtype=np.uint8)
    return np.array(img, dtype=np.uint8, order='C'), int(q[1:])
