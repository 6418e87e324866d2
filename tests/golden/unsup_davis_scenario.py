"""Seeded inputs of the unsupervised DAVIS 2017 post-processing fixture, shared by make_unsup_davis_golden.py (the
reference's ``limit_max_id`` on the CPU) and the tests (tests/test_unsup_davis17_{cpu,gpu}.py).

Every frame is regenerated from its seed (numpy PCG64), so the fixture stores only what ``limit_max_id`` wrote.
``run_case`` writes a case's inputs, calls ``limit(input_path, output_path, max_num_objects)`` and returns the error it
raised (type name, message) and a snapshot of the output tree: {relative path: (mode, sha256 of the palette, pixels)}.
"""
import hashlib
import os

import numpy as np
from PIL import Image

# video: (mode, frames, h, w, seed, layout, pool, extras)
#   layout 'rects': random rectangles with labels from pool, later ones covering earlier ones;
#          'stripes': every pool label as one vertical stripe of random width (each present in every frame);
#          'grid': a 5 x 8 grid of distinct labels, frame t taking pool[40 t : 40 t + 40].
#   extras: n (rectangles), tie (two labels of equal area drawn last), empty (all-zero frames),
#           late (first frame, label: a rectangle of an unseen label from that frame on), names ({frame: file name}).
R1, R2 = 0x010002, 0x020001  # R-major order puts R2 first; the saver's long-id order (R + 256 G + 65536 B) would not
BASE = {
    'bear': ('P', 9, 48, 64, 11, 'stripes', [1, 2, 3], dict(late=(7, 9))),
    'car': ('RGB', 5, 40, 56, 12, 'rects', [0x010005, 70000, 0x100007, 256, 255, 0xfffffe], dict(n=6, tie=(R1, R2))),
    'dog': ('L', 6, 32, 48, 13, 'rects', [10, 20, 30, 40, 200], dict(n=5, empty={0, 3}, names={5: '00005.PNG'})),
    'elk': ('RGBA', 4, 36, 44, 14, 'rects', list(range(0x200000, 0x200000 + 40 * 4099, 4099)), dict(n=30)),
    'fox': ('P', 12, 50, 70, 15, 'rects', list(range(1, 40)), dict(n=6, tie=(41, 42))),
    'zzz_empty': ('P', 0, 1, 1, 0, 'rects', [], {}),
}
DATASETS = {
    'base': BASE,
    'overflow': {
        'a': ('P', 3, 30, 40, 21, 'rects', [1, 2, 3, 4, 5, 6], dict(n=4)),
        'b': ('RGB', 8, 64, 80, 22, 'grid', list(range(1000, 1000 + 8 * 40)), {}),
        'c': ('P', 2, 30, 40, 23, 'rects', [1, 2], dict(n=2)),
    },
    'hd': {'hd': ('RGB', 2, 1080, 1920, 31, 'rects', list(range(0x300000, 0x300000 + 50 * 997, 997)), dict(n=30))},
}
# name: (dataset, max_num_objects, in place)
CASES = {
    'max20': ('base', 20, False),
    'max3': ('base', 3, False),
    'max1': ('base', 1, False),
    'max0': ('base', 0, False),
    'negative': ('base', -2, False),
    'overflow': ('overflow', 300, False),
    'hd': ('hd', 20, False),
    'in_place': ('base', 20, True),
}
INPUT_PALETTE = [(i * 53 + 7) % 256 for i in range(768)]  # the palette of the P inputs (not the output palette)


def frame_labels(video, t) -> np.ndarray:
    """int64 [h, w] labels of frame t."""
    mode, _, h, w, seed, layout, pool, extras = video
    rng = np.random.default_rng([seed, t])
    lab = np.zeros((h, w), np.int64)
    if t in extras.get('empty', ()):
        return lab
    if layout == 'stripes':
        cuts = np.sort(rng.choice(np.arange(1, w), len(pool) - 1, replace=False))
        for v, x0, x1 in zip(rng.permutation(pool), [0, *cuts], [*cuts, w]):
            lab[4:, x0:x1] = v
    elif layout == 'grid':
        cells = np.asarray(pool[40 * t:40 * t + 40]).reshape(5, 8)
        lab[:] = np.repeat(np.repeat(cells, -(-h // 5), 0), -(-w // 8), 1)[:h, :w]
    else:
        for v in rng.choice(pool, size=extras['n']):
            hh, ww = rng.integers(2, max(3, h // 2)), rng.integers(2, max(3, w // 2))
            y, x = rng.integers(0, h - hh + 1), rng.integers(0, w - ww + 1)
            lab[y:y + hh, x:x + ww] = v
    if 'tie' in extras:
        a, b = extras['tie']
        lab[h - 4:h - 1, 1:5] = a
        lab[h - 4:h - 1, 6:10] = b
    if 'late' in extras and t >= extras['late'][0]:
        lab[0:3, 0:5] = extras['late'][1]
    return lab


def frame_image(video, t) -> Image.Image:
    mode = video[0]
    lab = frame_labels(video, t)
    if mode in ('P', 'L'):
        img = Image.fromarray(lab.astype(np.uint8))
        if mode == 'P':
            img.putpalette(INPUT_PALETTE)
        return img
    rgb = [(lab >> 16) & 255, (lab >> 8) & 255, lab & 255]
    if mode == 'RGBA':
        rgb.append(np.random.default_rng([video[4], t, 1]).integers(0, 256, lab.shape))  # alpha carries no label
    return Image.fromarray(np.stack(rgb, -1).astype(np.uint8))  # RGB or RGBA by the channel count


def frame_name(video, t) -> str:
    return video[7].get('names', {}).get(t, f'{t:05d}.png')


def write_dataset(root, name) -> str:
    for vid, video in DATASETS[name].items():
        os.makedirs(os.path.join(root, vid), exist_ok=True)
        for t in range(video[1]):
            frame_image(video, t).save(os.path.join(root, vid, frame_name(video, t)))
    return root


def sha(data: bytes) -> str:
    return hashlib.sha256(data).hexdigest()


def snapshot(root):
    """{relative path: (mode, sha256 of the palette or None, pixels)} of every file under root."""
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            p = os.path.join(d, f)
            img = Image.open(p)
            out[os.path.relpath(p, root)] = (img.mode, sha(bytes(img.getpalette())) if img.mode == 'P' else None,
                                             np.array(img))
    return out


def assert_matches(meta, arrays, case, error, files):
    """The outcome of run_case equals the fixture's: the error, the set of files, and each file's mode, palette and
    pixels."""
    want = meta['cases'][case]
    assert (list(error) if error else None) == want['error'], (case, error)
    assert sorted(files) == sorted(want['files']), case
    for k, (mode, pal, px) in files.items():
        assert [mode, pal, sha(px.tobytes()), list(px.shape)] == want['files'][k], (case, k)
        if f'{case}/{k}' in arrays:
            np.testing.assert_array_equal(px, arrays[f'{case}/{k}'])


def run_case(limit, root, case):
    """-> ((error type name, message) or None, snapshot of the output tree)."""
    dataset, max_num_objects, in_place = CASES[case]
    src = write_dataset(os.path.join(root, 'in'), dataset)
    dst = src if in_place else os.path.join(root, 'out')
    error = None
    try:
        limit(src, dst, max_num_objects)
    except Exception as e:  # noqa: BLE001  (the fixture records which error, and where)
        error = (type(e).__name__, str(e))
    return error, snapshot(dst) if os.path.isdir(dst) else {}
