"""Folders, frames, detector fakes and the demo loop of the demo fixture (tests/golden/demo.{json,npz}).

Shared by make_demo_golden.py, which runs the UNMODIFIED reference's ``SimpleVideoReader``, ``get_input_frame_for_deva``,
processors and ``flush_buffer`` on the CPU, and by tests/test_demo_{cpu,gpu}.py, which run this package's drop-ins and
the same processors on the device.  Every file and frame is regenerated from seeds; nothing here needs a detector
package (the processors' imports are stubbed by detector_masks_scenario.install_detector_stubs).
"""
import hashlib
import os

import numpy as np
from PIL import Image

import detector_masks_scenario as dms

# the reader folder: name, (h, w), how it is written.  Sorted by name; the last file is not an image.
READER_FILES = [
    ('a_base420.jpg', (61, 83), dict(format='JPEG', quality=90, subsampling=2)),
    ('b_base444.jpg', (40, 57), dict(format='JPEG', quality=85, subsampling=0)),
    ('c_progressive.jpg', (33, 47), dict(format='JPEG', quality=90, progressive=True)),
    ('d_gray.jpg', (45, 38), dict(format='JPEG', quality=90, mode='L')),
    ('e_cmyk.jpg', (29, 41), dict(format='JPEG', quality=90, mode='CMYK')),
    ('f_rgb.png', (30, 44), dict(format='PNG')),
    ('g_rgba.png', (27, 35), dict(format='PNG', mode='RGBA')),
    ('h_notes.jpg', None, None),  # not an image: Pillow's UnidentifiedImageError at this index
    ('i_base420_large.jpg', (120, 161), dict(format='JPEG', quality=75)),
]

# the demo clip: 12 frames of 270x480 (short side not the demos' default 480, so the ingest resizes); frame 3 is a
# progressive and frame 7 a grayscale JPEG, which the device declines
CLIP_HW = (270, 480)
CLIP_FRAMES = 12
CLIP_SPECIAL = {3: dict(progressive=True), 7: dict(mode='L')}
DEMO_SIZE = 480

# get_input_frame_for_deva inputs: (h, w) of three small frames, each at these min_sides
INGEST_SHAPES = [(37, 53), (64, 48), (90, 61)]
INGEST_MIN_SIDES = [120, -1]

AUTO_MASK_SPEC = [('rand', 5)]
AUTO_SEED = 77
TEXT_BOXES = [(20, 30, 200, 150, 0.9, 0), (250, 60, 460, 250, 0.8, 1), (30, 160, 150, 260, 0.6, 0)]
PROMPT = 'cat.dog'
RUNS = [('auto', 'online'), ('auto', 'semionline'), ('text', 'online'), ('text', 'semionline')]


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def smooth(h, w, seed) -> np.ndarray:
    """A photo-like uint8 [h, w, 3] frame: a seeded 6x8 colour grid upsampled with Pillow's bilinear, plus a little noise
    (keeps every JPEG's coefficients where the device decoder accepts them)."""
    rng = np.random.default_rng(seed)
    grid = Image.fromarray(rng.integers(0, 256, (6, 8, 3), dtype=np.uint8)).resize((w, h), Image.BILINEAR)
    noise = rng.integers(-6, 7, (h, w, 3))
    return np.clip(np.asarray(grid).astype(np.int64) + noise, 0, 255).astype(np.uint8)


def _write(path, rgb, how):
    how = dict(how)
    fmt, mode = how.pop('format', 'JPEG'), how.pop('mode', 'RGB')
    Image.fromarray(rgb).convert(mode).save(path, fmt, **how)


def write_reader_folder(root):
    os.makedirs(root, exist_ok=True)
    for k, (name, hw, how) in enumerate(READER_FILES):
        p = os.path.join(root, name)
        if hw is None:
            open(p, 'wb').write(b'not an image, only its name says so\n')
        else:
            _write(p, smooth(*hw, seed=100 + k), how)
    return root


def clip_frame(t) -> np.ndarray:
    """Frame t of the demo clip: a fixed background with two blocks moving across it."""
    h, w = CLIP_HW
    img = smooth(h, w, seed=500).copy()
    img[40:120, 30 + 25 * t:130 + 25 * t] = (220, 60, 40)
    img[150:240, 400 - 20 * t:470 - 20 * t] = (40, 90, 200)
    return img


def write_demo_clip(root):
    os.makedirs(root, exist_ok=True)
    for t in range(CLIP_FRAMES):
        how = dict(format='JPEG', quality=90, **CLIP_SPECIAL.get(t, {}))
        _write(os.path.join(root, f'{t:05d}.jpg'), clip_frame(t), how)
    return root


def ingest_frame(h, w, k) -> np.ndarray:
    return np.random.default_rng(900 + k).integers(0, 256, (h, w, 3), dtype=np.uint8)


def read_items(reader, root):
    """The reader's items in order: [name, sha256 of the array, shape] or [name, error type, message] (``root``
    replaced by '<root>')."""
    out = []
    for i in range(len(reader)):
        try:
            a, p = reader[i]
            out.append([os.path.relpath(p, root), sha(a), list(a.shape)])
        except Exception as e:  # noqa: BLE001
            out.append([reader.frames[i], type(e).__name__, str(e).replace(root, '<root>')])
    return out


# ------------------------------------------------------------------------------------------------ the demo loop
def demo_config(base, kind, temporal):
    """The demo's config over the core's ``base``: detection every 5 frames, 3 voting frames (the demos' defaults)."""
    cfg = dict(base, size=DEMO_SIZE, temporal_setting=temporal, detection_every=5, num_voting_frames=3,
               max_missed_detection_count=10, max_num_objects=-1, suppress_small_objects=False,
               SAM_NUM_POINTS_PER_SIDE=dms.POINTS_PER_SIDE, SAM_OVERLAP_THRESHOLD=0.8)
    if kind == 'text':
        cfg.update(prompt=PROMPT, DINO_THRESHOLD=0.35, DINO_NMS_THRESHOLD=0.8)
    return cfg


def detectors(kind, device):
    """Fresh fakes for one run: (detector arguments of the processor, the fakes whose calls are recorded)."""
    if kind == 'auto':
        masks = dms.build_masks(AUTO_MASK_SPEC, *CLIP_HW, AUTO_SEED)
        sam = dms.FakeAutoSam(masks, dms.iou_preds(len(masks), AUTO_SEED), device)
        return (sam, ), [sam]
    gd, sam = dms.FakeGroundingDino(TEXT_BOXES, device), dms.FakeSamPredictor()
    return (gd, sam), [gd, sam]


def calls(fakes, with_points=True):
    """The fakes' recorded calls in order (the SAM generator's point prompts dropped unless ``with_points``)."""
    out = []
    for f in fakes:
        for c in f.calls:
            out.append(c if with_points or c[0] != 'generate' else c[:3] + [[a is not None for a in c[3]]])
    return out


class SaveRecorder:
    """A ResultSaver stand-in that records each save_mask call: frame name, shape, need_resize, the image's shape and
    SHA-256 and the prompts (``download`` turns a device image into the host array first)."""

    def __init__(self, download=None):
        self.calls, self.download = [], download

    def save_mask(self, prob, frame_name, need_resize=False, shape=None, save_the_mask=True, image_np=None,
                  prompts=None, path_to_image=None):
        img = image_np if self.download is None else self.download(image_np)
        self.calls.append([frame_name, [int(v) for v in shape], bool(need_resize), list(img.shape), sha(img),
                           prompts])


def run_demo(processors, flush_buffer, deva, frames, kind, saver, detector_args):
    """The demo scripts' loop: ``frames`` yields (frame, im_path); ``processors`` is the reference's
    automatic_processor or with_text_processor module."""
    deva.next_voting_frame = deva.config['num_voting_frames'] - 1
    deva.enabled_long_id()
    process = processors.process_frame_automatic if kind == 'auto' else processors.process_frame_with_text
    for ti, (frame, im_path) in enumerate(frames):
        process(deva, *detector_args, im_path, saver, ti, image_np=frame)
    flush_buffer(deva, saver)
