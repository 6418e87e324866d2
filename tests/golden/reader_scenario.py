"""Seeded clips for the dataset readers (deva/inference/data/) and the runs that read them.

``clip_files()`` builds every clip's files as bytes (stored in readers.npz, so a test reads the very files the fixture
was made from): small frames at 96x160, portrait 161x97 and 17x9 in 4:2:0 / 4:2:2 / 4:4:4 JPEG, JPEGs the device
declines (progressive, greyscale, Exif), masks as P with a palette, L, RGB ids above 255, RGBA, 16-bit, interlaced and
missing, soft prob folders (with a ``.csv`` entry), per-frame detection JSONs, and the real bmx-trees and vipseg
frames and masks of tests/golden/ (read from their own files there, ``REAL``).  ``RUNS`` names each reader run: (name,
reader class, clip, keyword arguments).  ``record`` turns one collated item into JSON structure and arrays.
"""
import hashlib
import io
import os
import struct
import zlib

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT_TOKEN = '<root>'


def _jpeg(rgb, **kw):
    b = io.BytesIO()
    Image.fromarray(rgb).save(b, 'JPEG', quality=90, **kw)
    return b.getvalue()


def _png(img):
    b = io.BytesIO()
    img.save(b, 'PNG')
    return b.getvalue()


def _interlaced_png(index):
    """An Adam7-interlaced 8-bit grey PNG (Pillow writes no interlaced files), zlib-compressed by hand."""
    h, w = index.shape
    starts = ((0, 0, 8, 8), (0, 4, 8, 8), (4, 0, 8, 4), (0, 2, 4, 4), (2, 0, 4, 2), (0, 1, 2, 2), (1, 0, 2, 1))
    raw = b''
    for y0, x0, dy, dx in starts:
        sub = index[y0::dy, x0::dx]
        if sub.size:
            raw += b''.join(b'\0' + row.tobytes() for row in sub)

    def chunk(kind, data):
        return struct.pack('>I', len(data)) + kind + data + struct.pack('>I', zlib.crc32(kind + data))
    return (b'\x89PNG\r\n\x1a\n' + chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, 8, 0, 0, 0, 1)) +
            chunk(b'IDAT', zlib.compress(raw)) + chunk(b'IEND', b''))


def _frame(rng, h, w):
    """A smooth random RGB frame (blocky noise upsampled), so JPEG artefacts stay realistic."""
    small = rng.integers(0, 256, (max(h // 8, 1) + 1, max(w // 8, 1) + 1, 3)).astype(np.uint8)
    return np.asarray(Image.fromarray(small).resize((w, h), Image.BILINEAR))


def _index(rng, h, w, k):
    m = np.zeros((h, w), np.uint8)
    for o in range(1, k + 1):
        y, x = rng.integers(0, h), rng.integers(0, w)
        m[max(0, y - h // 4):y + h // 4, max(0, x - w // 4):x + w // 4] = o
    return m


def _palette_png(index):
    im = Image.frombytes('P', index.shape[::-1], index.tobytes())
    im.putpalette([v for i in range(256) for v in ((i * 37) % 256, (i * 91) % 256, (i * 53) % 256)])
    return _png(im)


def clip_files(seed=0):
    """{relative path: bytes} of every clip."""
    rng = np.random.default_rng(seed)
    f = {}
    # vos: 96x160, one frame per subsampling, then the declined JPEGs; masks of every kind, one frame without
    h, w = 96, 160
    subs = (2, 1, 0, 2, 2, 2, 2)
    for t, sub in enumerate(subs):
        rgb = _frame(rng, h, w)
        if t == 4:
            data = _jpeg(rgb, progressive=True)
        elif t == 5:
            data = _jpeg(np.asarray(Image.fromarray(rgb).convert('L')))
        elif t == 6:
            exif = Image.Exif()
            exif[0x010F] = 'deva'
            data = _jpeg(rgb, exif=exif.tobytes())
        else:
            data = _jpeg(rgb, subsampling=sub)
        f[f'vos/JPEGImages/{t:05d}.jpg'] = data
        idx = _index(rng, h, w, 3)
        if t in (0, 6):
            f[f'vos/Annotations/{t:05d}.png'] = _palette_png(idx)
        elif t == 1:
            f[f'vos/Annotations/{t:05d}.png'] = _png(Image.fromarray(idx * 40))
        elif t == 3:
            f[f'vos/Annotations/{t:05d}.png'] = _png(Image.fromarray(np.dstack([idx * 50] * 3 + [np.full_like(idx, 255)])))
        elif t == 4:
            f[f'vos/Annotations/{t:05d}.png'] = _png(Image.fromarray(idx.astype(np.uint16) * 300))
        elif t == 5:
            f[f'vos/Annotations/{t:05d}.png'] = _interlaced_png(idx)
        # t == 2 has no mask
    # shapes for size_dir: the same names, frames at another size
    for t in range(len(subs)):
        f[f'vos/Sizes/{t:05d}.jpg'] = _jpeg(_frame(rng, 120, 200))
    # portrait and tiny clips
    for name, (h2, w2) in (('portrait', (161, 97)), ('tiny', (17, 9))):
        for t in range(3):
            f[f'{name}/JPEGImages/{t:05d}.jpg'] = _jpeg(_frame(rng, h2, w2), subsampling=(2, 1, 0)[t])
            f[f'{name}/Annotations/{t:05d}.png'] = _palette_png(_index(rng, h2, w2, 2))
    # soft masks: prob folders (and a csv), single-object folder
    for t in range(3):
        f[f'soft/JPEGImages/{t:05d}.jpg'] = _jpeg(_frame(rng, 96, 160))
        for obj in ('obj1', 'obj2'):
            prob = np.ascontiguousarray(_frame(rng, 96, 160)[..., 0])
            f[f'soft/Probs/{obj}/{t:05d}.png'] = _png(Image.fromarray(prob))
        f[f'soft/Single/{t:05d}.png'] = _png(Image.fromarray(np.ascontiguousarray(_frame(rng, 96, 160)[..., 1])))
    f['soft/Probs/stats.csv'] = b'object,area\nobj1,1\n'
    # detections: P, L, RGB ids > 255, missing; JSONs on some frames
    for t in range(5):
        f[f'det/JPEGImages/{t:05d}.jpg'] = _jpeg(_frame(rng, 96, 160))
        idx = _index(rng, 96, 160, 4)
        if t in (0, 3):
            f[f'det/Masks/{t:05d}.png'] = _palette_png(idx)
        elif t == 1:
            f[f'det/Masks/{t:05d}.png'] = _png(Image.fromarray(idx * 9))
        elif t == 2:
            ids = idx.astype(np.int64) * 70001 + 3
            f[f'det/Masks/{t:05d}.png'] = _png(Image.fromarray(
                np.dstack([ids % 256, ids // 256 % 256, ids // 65536 % 256]).astype(np.uint8)))
        if t % 2 == 0:
            f[f'det/Masks/{t:05d}.json'] = f'{{"frame": {t}}}'.encode()
    # a detection clip whose first frame has no mask: is_rgb stays None
    f['det_none/JPEGImages/00000.jpg'] = _jpeg(_frame(rng, 96, 160))
    f['det_none/Masks/00001.png'] = _palette_png(_index(rng, 96, 160, 2))
    f['det_none/JPEGImages/00001.jpg'] = _jpeg(_frame(rng, 96, 160))
    return f


# the real frames and masks, read from their files in tests/golden (not stored again in readers.npz)
REAL = {f'{clip}/{kind}/00000.{ext}': f'{prefix}_{stem}.{ext}'
        for clip, stem in (('bmx', 'davis_bmx-trees_00000'), ('vipseg', 'vipseg_00001255'))
        for kind, ext, prefix in (('JPEGImages', 'jpg', 'jpeg_decode'), ('Annotations', 'png', 'png_decode'))}


def real_files():
    """{relative path: bytes} of the real clips."""
    return {rel: open(os.path.join(HERE, name), 'rb').read() for rel, name in REAL.items()}


def stored_files(z):
    """{relative path: bytes} of every clip: the synthetic ones from readers.npz ``z``, the real ones from their files."""
    files = {k[len('file/'):]: z[k].tobytes() for k in z.files if k.startswith('file/')}
    files.update(real_files())
    return files


RUNS = []
for _size in (-1, 240, 480):
    RUNS += [(f'vos_first_{_size}', 'VideoReader', 'vos', dict(size=_size)),
             (f'vos_all_{_size}', 'VideoReader', 'vos', dict(size=_size, use_all_masks=True))]
RUNS += [
    ('vos_start_end', 'VideoReader', 'vos', dict(size=240, start=1, end=5, use_all_masks=True)),
    ('vos_sampled', 'VideoReader', 'vos', dict(size=-1, num_sampled_frames=3)),
    ('vos_reverse', 'VideoReader', 'vos', dict(size=240, reverse=True, use_all_masks=True)),
    ('vos_to_save', 'VideoReader', 'vos', dict(size=-1, to_save=['00001', '00003'])),
    ('vos_enabled', 'VideoReader', 'vos', dict(size=240, enabled_frame_list=['00000', '00002', '00003'])),
    ('vos_size_dir', 'VideoReader', 'vos', dict(size=240, size_dir='Sizes', use_all_masks=True)),
    ('portrait_240', 'VideoReader', 'portrait', dict(size=240, use_all_masks=True)),
    ('portrait_-1', 'VideoReader', 'portrait', dict(size=-1, use_all_masks=True)),
    ('tiny_480', 'VideoReader', 'tiny', dict(size=480, use_all_masks=True)),
    ('soft_multi_240', 'VideoReader', 'soft', dict(size=240, soft_mask=True, use_all_masks=True)),
    ('soft_multi_-1', 'VideoReader', 'soft', dict(size=-1, soft_mask=True)),
    ('soft_object_480', 'VideoReader', 'soft', dict(size=480, soft_mask=True, object_name='obj2')),
    ('soft_single_240', 'VideoReader', 'soft', dict(size=240, soft_mask=True, multi_object=False,
                                                    use_all_masks=True)),
    ('bmx_240', 'VideoReader', 'bmx', dict(size=240)),
    ('bmx_480', 'VideoReader', 'bmx', dict(size=480)),
    ('vipseg_480', 'VideoReader', 'vipseg', dict(size=480)),
    ('det_-1', 'DetectionVideoReader', 'det', dict(size=-1)),
    ('det_480', 'DetectionVideoReader', 'det', dict(size=480)),
    ('det_start_end', 'DetectionVideoReader', 'det', dict(size=480, start=1, end=3)),
    ('det_none', 'DetectionVideoReader', 'det_none', dict(size=-1)),
    ('det_reverse', 'DetectionVideoReader', 'det', dict(size=-1, reverse=True)),
    ('det_vipseg', 'DetectionVideoReader', 'vipseg', dict(size=480)),
]
MASK_DIRS = {'vos': 'Annotations', 'portrait': 'Annotations', 'tiny': 'Annotations', 'bmx': 'Annotations',
             'vipseg': 'Annotations', 'soft_single': 'Single', 'soft': 'Probs', 'det': 'Masks', 'det_none': 'Masks'}


def materialise(files, root):
    """Writes the clips under ``root``."""
    for rel, data in files.items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, 'wb') as fh:
            fh.write(bytes(data))


def make_reader(classes, run, root):
    """The run's reader, ``classes`` mapping 'VideoReader' / 'DetectionVideoReader' to the implementation."""
    name, cls, clip, kw = run
    kw = dict(kw)
    mask_dir = MASK_DIRS['soft_single' if kw.get('multi_object') is False else clip]
    if 'size_dir' in kw:
        kw['size_dir'] = os.path.join(root, clip, kw['size_dir'])
    return classes[cls](clip, os.path.join(root, clip, 'JPEGImages'), os.path.join(root, clip, mask_dir), **kw)


FULL = 1 << 14  # tensors up to this many elements are stored whole; larger ones (float frames) as a digest


def digest(t) -> str:
    return hashlib.sha256(np.ascontiguousarray(t.numpy()).tobytes()).hexdigest()


def record(value, root, prefix, arrays):
    """JSON structure of a collated item (tensors as dtype / shape / array key, strings with ``root`` replaced);
    tensors go to ``arrays``.  A tensor over ``FULL`` elements is kept as the sha256 of its bytes, with its float64
    sum to tell how far a mismatch is."""
    if isinstance(value, dict):
        return {'dict': [[k, record(v, root, f'{prefix}/{k}', arrays)] for k, v in value.items()]}
    if isinstance(value, (list, tuple)):
        return {type(value).__name__: [record(v, root, f'{prefix}/{i}', arrays) for i, v in enumerate(value)]}
    if isinstance(value, str):
        return {'str': value.replace(root, ROOT_TOKEN)}
    if torch.is_tensor(value):
        t = value.detach().cpu()
        rec = {'tensor': str(t.dtype), 'shape': list(t.shape)}
        if t.numel() > FULL:
            rec.update(sha256=digest(t), sum=float(t.double().sum()))
        else:
            rec['key'] = prefix
            arrays[prefix] = t.contiguous().numpy()
        return rec
    return {type(value).__name__: value}


def error_record(e, root):
    return {'error': type(e).__name__, 'message': str(e).replace(root, ROOT_TOKEN)}
