"""Scripted result-saver sessions shared by make_saver_golden.py (the reference's ResultSaver on the CPU) and
tests/test_result_saver_gpu.py (this package's ResultSaver on the GPU).

Probabilities and frames are regenerated from per-frame seeds (numpy PCG64), so the fixture stores only the seeds and
what the savers produced.  Third-party outputs are captured by recorders instead of encoders: ``PIL.Image.Image.save``
records (relative path, mode, palette, pixels), ``pycocotools.mask.encode`` and ``supervision`` are stubs that record
their arguments, and the gradio writer records its frames.
"""
import contextlib
import hashlib
import os
import sys
import types

import numpy as np
from PIL import Image

SRC = (240, 427)  # the step's resolution
OUT = (270, 481)  # the original resolution the driver resizes back to

# dataset, use_long_id, video_name, palette, frames: (ops before save_mask, save_mask keyword arguments)
# ops: ('add', [(id, category_id, score), ...]) or ('del', [id, ...]); kwargs 'resize' / 'image' / 'path' are
# expanded by drive(): resize -> need_resize (positional when 'positional') and shape, image -> image_np, path ->
# path_to_image of the frame written as PNG.
PALETTE = [(i * 37) % 256 for i in range(768)]
SESSIONS = [
    ('vipseg', False, 'vid_a', PALETTE, [
        ([('add', [(5, 1, 0.9), (9, 2, 0.8)])], dict(resize=True)),
        ([('add', [(12, 0, 0.7)])], dict(resize='positional')),
        ([('del', [9])], dict(resize=True)),
    ]),
    ('burst', False, 'ds/seq_b', None, [
        ([('add', [(3, 1, 0.5), (7, 2, 0.6)])], dict(resize=True)),
        ([('add', [(11, 0, 0.4)]), ('del', [3])], dict(resize=True)),
    ]),
    ('unsup_davis17', False, 'v_c', PALETTE, [
        ([('add', [(1, None, None), (2, None, None)])], dict()),
        ([('del', [1]), ('add', [(4, None, None)])], dict(resize=False)),
    ]),
    ('ref_davis', False, 'v_d', PALETTE, [
        ([('add', [(1, None, None)])], dict(resize='positional_false')),
        ([('add', [(2, None, None)])], dict()),
    ]),
    ('demo', True, None, None, [
        ([('add', [(300, 0, 0.9), (70000, 1, 0.8), (1234567, 2, 0.75)])], dict(resize=True, image=True,
                                                                               prompts=True)),
        ([('add', [(4096, 1, 0.6)])], dict(resize=True, image=True, save_the_mask=False)),
        ([], dict(resize=True, path=True, prompts=True)),
        ([('del', [70000])], dict(resize=True, image=True)),
        ([('add', [(500, 2, 0.55)])], dict(resize=True, image=True, prompts=True)),
    ]),
    ('demo', False, None, None, [
        ([('add', [(8, 0, 0.9), (13, 1, 0.3)])], dict(resize=True, image=True)),
        ([('del', [8])], dict(resize=True, image=True)),
    ]),
    ('gradio', True, None, None, [
        ([('add', [(777, 0, 0.9), (65536, 1, 0.8)])], dict(resize=True, image=True, prompts=True)),
        ([('del', [777]), ('add', [(1000, 2, 0.5)])], dict(resize=True, image=True, prompts=True)),
    ]),
    # longer than the product's ring of pinned buffers (12 slots), objects changing while frames are queued
    ('vipseg', False, 'vid_long', None, [
        ([('add', [(20 + t, t % 3, 0.5 + 0.02 * t)])] + ([('del', [20 + t - 3])] if t % 4 == 3 else []),
         dict(resize=True)) for t in range(16)
    ]),
]
PROMPTS = ['person', 'dog', 'kite']


def make_prob(seed: int, c: int) -> np.ndarray:
    """float32 [c, *SRC]: per-channel background levels (channel 0 leads) overlaid by one rectangle per object in which
    that object leads; later rectangles cover earlier ones, so an object can vanish (zero area)."""
    rng = np.random.default_rng(seed)
    h, w = SRC
    p = np.empty((c, h, w), np.float32)
    bg = rng.uniform(0, 0.2, c)
    bg[0] += 0.6
    p[:] = bg[:, None, None]
    for k in range(1, c):
        hh, ww = rng.integers(30, 120), rng.integers(40, 200)
        y0, x0 = rng.integers(0, h - hh), rng.integers(0, w - ww)
        lv = rng.uniform(0, 0.2, c)
        lv[k] += 0.7
        p[:, y0:y0 + hh, x0:x0 + ww] = lv[:, None, None]
    return p


def make_image(seed: int, shape) -> np.ndarray:
    """uint8 [*shape, 3]: random 16x16 colour tiles (they keep the recorded overlays compressible)."""
    h, w = shape
    tiles = np.random.default_rng(seed).integers(0, 256, (h // 16 + 1, w // 16 + 1, 3), dtype=np.uint8)
    return np.ascontiguousarray(tiles.repeat(16, 0).repeat(16, 1)[:h, :w])


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


class Recorder:
    """Installs the recording stubs; ``events`` lists everything recorded, in order."""

    def __init__(self):
        self.events = []
        self.root = None

    @contextlib.contextmanager
    def installed(self):
        rec = self
        orig_save = Image.Image.save

        def save(img, fp, *a, **k):
            rel = os.path.relpath(fp, rec.root)
            pal = img.getpalette() if img.mode == 'P' else None
            rec.events.append(('image', rel, img.mode, pal, np.array(img)))

        coco = types.ModuleType('pycocotools')
        coco.mask = types.ModuleType('pycocotools.mask')

        def encode(m):
            rec.events.append(('rle', bool(m.flags['F_CONTIGUOUS']), m.dtype.str, np.array(m)))
            return {'size': list(m.shape), 'counts': f'{int(m.sum())}:{digest(np.packbits(m))}'.encode()}

        coco.mask.encode = encode
        sv = types.ModuleType('supervision')

        class Detections:
            def __init__(self, xyxy, confidence=None, class_id=None):
                self.xyxy, self.confidence, self.class_id = xyxy, confidence, class_id
                rec.events.append(('detections', np.asarray(xyxy).dtype.str, np.asarray(xyxy).tolist(),
                                   np.asarray(confidence).tolist(), np.asarray(class_id).tolist()))

        class BoundingBoxAnnotator:
            def annotate(self, scene, detections):
                rec.events.append(('boxes', np.array(scene)))
                return scene

        class LabelAnnotator:
            def annotate(self, scene, detections, labels=None):
                rec.events.append(('labels', list(labels)))
                return scene

        sv.Detections, sv.BoundingBoxAnnotator, sv.LabelAnnotator = Detections, BoundingBoxAnnotator, LabelAnnotator
        saved = {k: sys.modules.get(k) for k in ('pycocotools', 'pycocotools.mask', 'supervision')}
        sys.modules.update({'pycocotools': coco, 'pycocotools.mask': coco.mask, 'supervision': sv})
        Image.Image.save = save
        try:
            yield orig_save
        finally:
            Image.Image.save = orig_save
            for k, v in saved.items():
                if v is None:
                    sys.modules.pop(k, None)
                else:
                    sys.modules[k] = v


class Writer:
    def __init__(self, rec: Recorder):
        self.rec = rec

    def write(self, frame):
        self.rec.events.append(('gradio', np.array(frame)))


def drive(ResultSaver, ObjectManager, ObjectInfo, session, seeds, root, rec: Recorder, orig_save, to_prob=None):
    """Runs one session through ``ResultSaver``; returns its video_json (or None).  ``seeds[t]`` = (prob seed, image
    seed) of frame t; ``to_prob`` moves the float32 tensor where the saver expects it (identity for the reference)."""
    import torch
    dataset, long_id, video, palette, frames = session
    np.random.seed(0)
    om = ObjectManager()
    om.use_long_id = long_id
    rec.root = root
    saver = ResultSaver(root, video, dataset=dataset, object_manager=om, palette=palette)
    if dataset == 'gradio':
        saver.writer = Writer(rec)
    for t, (ops, kw) in enumerate(frames):
        for op, arg in ops:
            if op == 'add':
                om.add_new_objects([ObjectInfo(i, category_id=c, score=s) for i, c, s in arg])
            else:
                om.delete_object(arg)
        prob_seed, image_seed = seeds[t]
        prob = torch.from_numpy(make_prob(prob_seed, om.num_obj + 1))
        if to_prob is not None:
            prob = to_prob(prob)
        resize = kw.get('resize', False)
        shape = OUT if resize in (True, 'positional') else SRC
        args, kwargs = [prob, f'{t:05d}.jpg'], {}
        if resize == 'positional':
            args.append(True)
            kwargs['shape'] = OUT
        elif resize == 'positional_false':
            args.append(False)
        elif resize:
            kwargs.update(need_resize=True, shape=OUT)
        if 'save_the_mask' in kw:
            kwargs['save_the_mask'] = kw['save_the_mask']
        image = make_image(image_seed, shape)
        if kw.get('image'):
            kwargs['image_np'] = image
        if kw.get('path'):
            p = os.path.join(root, f'input_{t}.png')
            orig_save(Image.fromarray(image), p)
            kwargs['path_to_image'] = p
        if kw.get('prompts'):
            kwargs['prompts'] = PROMPTS
        saver.save_mask(*args, **kwargs)
    saver.end()
    return getattr(saver, 'video_json', None)
