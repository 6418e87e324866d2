"""Cases and detector fakes of the detector-mask fixture (tests/golden/detector_masks.{json,npz}).

Shared by make_detector_masks_golden.py, which runs the UNMODIFIED reference ``auto_segment`` / ``segment_with_text``
on the CPU with these fakes in place of SAM and Grounding-DINO, and by the tests, which run this package's drop-ins
with the same fakes and compare maps, segment lists and the calls each fake recorded.  Masks are regenerated from the
case specs and seeds; nothing here needs a detector package.
"""
import sys
import types
import zlib

import numpy as np
import torch

IMAGE_SEED = 5


def image(h, w, seed=IMAGE_SEED):
    return np.random.default_rng(seed + h * 7 + w).integers(0, 256, (h, w, 3), dtype=np.uint8)


def checksum(a) -> int:
    return zlib.crc32(np.ascontiguousarray(a).tobytes())


# ------------------------------------------------------------------------------------------------ automatic path
def build_masks(spec, h, w, seed):
    """spec: list of ('rand', count) | ('rect', y0, x0, y1, x1) | ('dup', i) | ('nest', i) | ('pixel', y, x) | ('empty',)
    -> bool [n, h, w]."""
    rng = np.random.default_rng(seed)
    out = []
    yy, xx = np.mgrid[0:h, 0:w]
    for op in spec:
        if op[0] == 'rand':
            for _ in range(op[1]):
                m = np.zeros((h, w), bool)
                cy, cx = rng.integers(0, h), rng.integers(0, w)
                ry, rx = rng.integers(1, max(2, h // 3)), rng.integers(1, max(2, w // 3))
                if rng.random() < 0.5:
                    m[max(0, cy - ry):cy + ry, max(0, cx - rx):cx + rx] = True
                else:
                    m |= ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1
                out.append(m)
        elif op[0] == 'rect':
            m = np.zeros((h, w), bool)
            m[op[1]:op[3], op[2]:op[4]] = True
            out.append(m)
        elif op[0] == 'dup':
            out.append(out[op[1]].copy())
        elif op[0] == 'nest':
            ys, xs = np.nonzero(out[op[1]])
            m = np.zeros((h, w), bool)
            y0, y1, x0, x1 = ys.min(), ys.max() + 1, xs.min(), xs.max() + 1
            m[y0 + (y1 - y0) // 4:y1 - (y1 - y0) // 4, x0 + (x1 - x0) // 4:x1 - (x1 - x0) // 4] = True
            out.append(m & out[op[1]])
        elif op[0] == 'pixel':
            m = np.zeros((h, w), bool)
            m[op[1], op[2]] = True
            out.append(m)
        else:
            out.append(np.zeros((h, w), bool))
    return np.stack(out) if out else np.zeros((0, h, w), bool)


def forward_mask(kind, h, w):
    if kind is None:
        return None
    m = torch.zeros((h, w), dtype=torch.int64)
    if kind == 'all':
        m[:] = 3
    elif kind == 'left':
        m[:, :w // 2] = 1
    return m


# name, (h, w), min_side, suppress, threshold, forward kind, mask spec
AUTO_CASES = [
    ('empty_stack', (48, 64), 24, True, 0.8, None, []),
    ('one_mask', (48, 64), 24, True, 0.8, None, [('rand', 1)]),
    ('one_mask_free', (48, 64), 24, False, 0.8, None, [('rand', 1)]),
    ('overlap_nested_dup', (90, 120), 60, True, 0.6, None, [('rand', 6), ('nest', 0), ('nest', 2), ('dup', 1),
                                                            ('rand', 3), ('dup', 5)]),
    ('overlap_nested_dup_free', (90, 120), 60, False, 0.6, None, [('rand', 6), ('nest', 0), ('dup', 1), ('rand', 3)]),
    ('vanishing_pixel', (96, 128), 32, True, 0.5, None, [('rand', 3), ('pixel', 41, 51), ('rand', 2)]),
    ('threshold_rejects', (101, 77), 60, True, 0.9, None, [('rand', 12)]),
    ('f32_boundary', (40, 50), 0, True, 0.69999999, None, [('rect', 0, 0, 30, 40), ('rect', 29, 37, 31, 42)]),
    ('free_id_channel_mismatch', (40, 50), 0, False, 0.8, None, [('empty',), ('rect', 5, 5, 20, 30), ('empty',),
                                                                ('rect', 10, 10, 35, 45)]),
    ('same_size', (37, 53), 0, True, 0.7, None, [('rand', 8), ('dup', 2)]),
    ('same_size_free', (37, 53), -1, False, 0.7, None, [('rand', 8)]),
    ('upscale_odd', (33, 47), 70, True, 0.7, None, [('rand', 7), ('dup', 0)]),
    ('upscale_odd_free', (33, 47), 70, False, 0.7, None, [('rand', 7)]),
    ('hd_to_480', (1080, 1920), 480, True, 0.8, None, [('rand', 40), ('dup', 3)]),
    ('hd_to_480_free', (1080, 1920), 480, False, 0.8, None, [('rand', 40)]),
    ('forward_points', (64, 96), 48, True, 0.8, 'left', [('rand', 5)]),
    ('forward_no_points', (64, 96), 48, True, 0.8, 'all', [('rand', 5)]),
]
POINTS_PER_SIDE = 8


def auto_config(threshold):
    return {'SAM_NUM_POINTS_PER_SIDE': POINTS_PER_SIDE, 'SAM_OVERLAP_THRESHOLD': threshold}


class FakeAutoSam:
    """SamAutomaticMaskGenerator stand-in: returns a fixed mask stack (bool, on `device`) and records generate()."""

    def __init__(self, masks, iou_preds, device):
        self.predictor = types.SimpleNamespace(device=torch.device(device))
        self.masks = torch.from_numpy(masks).to(device)
        self.iou_preds = torch.from_numpy(iou_preds).to(device)
        self.calls = []

    def generate(self, image, *args):
        self.calls.append(['generate', list(image.shape), checksum(image),
                           [None if a is None else np.asarray(a, np.float64).tolist() for a in args]])
        return {'masks': self.masks, 'iou_preds': self.iou_preds}


def iou_preds(n, seed):
    return np.random.default_rng(seed + 1).uniform(0.5, 1.0, n).astype(np.float32)


# ------------------------------------------------------------------------------------------------ text path
class Detections:
    """supervision.Detections stand-in: the fields segment_with_text touches, with `area` as mask pixel counts."""

    def __init__(self, xyxy, confidence, class_id):
        self.xyxy, self.confidence, self.class_id, self.mask = xyxy, confidence, class_id, None

    @property
    def area(self):
        return np.array([np.sum(m) for m in self.mask])


# name, (h, w), min_side, nms threshold, boxes [(x0, y0, x1, y1, confidence, class id)]
TEXT_CASES = [
    ('no_boxes', (48, 64), 24, 0.8, []),
    ('nms_suppression', (96, 128), 48, 0.5, [(10, 10, 60, 50, 0.9, 0), (12, 11, 61, 52, 0.8, 1),
                                             (70, 40, 120, 90, 0.7, 1)]),
    ('equal_areas', (96, 128), 48, 0.8, [(5, 5, 45, 35, 0.6, 0), (60, 50, 100, 80, 0.7, 0),
                                         (20, 30, 60, 60, 0.5, 2)]),
    ('empty_after_resize', (135, 240), 60, 0.8, [(100, 50, 101, 51, 0.9, 0), (10, 10, 200, 120, 0.8, 1),
                                                 (50, 60, 51, 61, 0.7, 1), (30, 20, 90, 70, 0.6, 2)]),
    ('none_class_ids', (96, 128), 48, 0.8, [(10, 10, 70, 60, 0.9, None), (40, 30, 110, 90, 0.8, 3),
                                            (0, 0, 128, 96, 0.3, None)]),
    ('exact_2x_down', (96, 128), 48, 0.8, [(7, 9, 63, 77, 0.9, 0), (33, 21, 101, 90, 0.8, 1), (50, 5, 127, 40, 0.7, 2)]),
    ('same_size_odd', (37, 53), 0, 0.8, [(3, 4, 30, 25, 0.9, 0), (10, 10, 50, 35, 0.8, 1)]),
    ('hd_to_480', (1080, 1920), 480, 0.8, [(100 + 90 * i, 50 + 40 * i, 600 + 70 * i, 500 + 30 * i, 0.9 - 0.04 * i, i % 3)
                                           for i in range(12)]),
]
TEXT_CONFIG = {'DINO_THRESHOLD': 0.35}


def text_config(nms):
    return dict(TEXT_CONFIG, DINO_NMS_THRESHOLD=nms)


class FakeGroundingDino:
    def __init__(self, boxes, device):
        self.device = device
        self.boxes = boxes
        self.calls = []

    def predict_with_classes(self, image, classes, box_threshold, text_threshold):
        self.calls.append(['predict_with_classes', list(image.shape), checksum(image), list(classes), box_threshold,
                           text_threshold])
        b = self.boxes
        xyxy = np.array([x[:4] for x in b], np.float32).reshape(-1, 4)
        conf = np.array([x[4] for x in b], np.float32)
        ids = [x[5] for x in b]
        cls = np.array(ids, dtype=object) if any(i is None for i in ids) else np.array(ids, dtype=np.int64)
        return Detections(xyxy, conf, cls)


class FakeSamPredictor:
    """SamPredictor stand-in: three nested box masks per box; scores seeded by the box's size, so equal-size boxes pick
    the same inset (equal areas)."""

    def __init__(self):
        self.calls = []
        self.hw = None

    def set_image(self, image, image_format='RGB'):
        self.hw = image.shape[:2]
        self.calls.append(['set_image', list(image.shape), checksum(image), image_format])

    def predict(self, box, multimask_output):
        self.calls.append(['predict', np.asarray(box, np.float64).tolist(), multimask_output])
        h, w = self.hw
        x0, y0, x1, y1 = [int(round(float(v))) for v in box]
        masks = np.zeros((3, h, w), bool)
        for j in range(3):
            a, b = min(y0 + j, y1 - 1), min(x0 + 2 * j, x1 - 1)
            masks[j, a:max(a + 1, y1 - j), b:max(b + 1, x1 - j)] = True
        scores = np.random.default_rng((x1 - x0) * 1000 + (y1 - y0)).random(3).astype(np.float32)
        return masks, scores, None


# ------------------------------------------------------------------------------------------------ reference loading
def install_detector_stubs(recorder):
    """Stub modules for segment_anything, groundingdino and deva.ext.SAM / MobileSAM / LightHQSAM.  Model builders
    record their calls in ``recorder`` (a list) and return recording models."""

    class Model:
        def __init__(self, name):
            self.name = name

        def load_state_dict(self, sd, strict):
            recorder.append(['load_state_dict', self.name, sd, strict])

        def to(self, device):
            recorder.append(['to', self.name, str(device)])
            return self

    def builder(name):
        def build(*args, **kwargs):
            recorder.append([name, list(args), sorted(kwargs.items())])
            return Model(name)
        return build

    class Registry:
        def __init__(self, name):
            self.name = name

        def __getitem__(self, version):
            return builder(f'{self.name}[{version}]')

    class Generator:
        def __init__(self, model, **kwargs):
            recorder.append(['SamAutomaticMaskGenerator', model.name, sorted(kwargs.items())])

    class Predictor:
        def __init__(self, model):
            recorder.append(['SamPredictor', model.name])
            self.name = model.name

    class GDModel:
        def __init__(self, **kwargs):
            recorder.append(['GroundingDINOModel', sorted(kwargs.items())])

    def module(name, **attrs):
        m = types.ModuleType(name)
        m.__path__ = []
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    module('segment_anything', sam_model_registry=Registry('sam_model_registry'), SamPredictor=Predictor,
           sam_hq_model_registry=Registry('sam_hq_model_registry'), SamAutomaticMaskGenerator=Generator)
    module('groundingdino')
    module('groundingdino.util')
    module('groundingdino.util.inference', Model=GDModel)
    for pkg, sub, attr, name in (('deva.ext.SAM', 'automatic_mask_generator', 'SamAutomaticMaskGenerator', None),
                                 ('deva.ext.MobileSAM', 'setup_mobile_sam', 'setup_model', 'setup_mobile_sam'),
                                 ('deva.ext.LightHQSAM', 'setup_light_hqsam', 'setup_model', 'setup_light_hqsam')):
        module(pkg)
        module(f'{pkg}.{sub}', **{attr: Generator if name is None else builder(name)})


MODEL_CONFIGS = [
    {'sam_variant': 'mobile', 'MOBILE_SAM_CHECKPOINT_PATH': 'm.pt', 'SAM_NUM_POINTS_PER_SIDE': 16,
     'SAM_NUM_POINTS_PER_BATCH': 32, 'SAM_PRED_IOU_THRESHOLD': 0.88},
    {'sam_variant': 'Original', 'SAM_ENCODER_VERSION': 'vit_b', 'SAM_CHECKPOINT_PATH': 's.pth',
     'SAM_NUM_POINTS_PER_SIDE': 64, 'SAM_NUM_POINTS_PER_BATCH': 64, 'SAM_PRED_IOU_THRESHOLD': 0.8},
]
GD_CONFIGS = [dict(c, GROUNDING_DINO_CONFIG_PATH='g.py', GROUNDING_DINO_CHECKPOINT_PATH='g.pth',
                   HQ_SAM_CHECKPOINT_PATH='hq.pth', LIGHT_HQ_SAM_CHECKPOINT_PATH='lhq.pth')
              for c in MODEL_CONFIGS + [{'sam_variant': 'sam_hq', 'SAM_ENCODER_VERSION': 'vit_l'},
                                        {'sam_variant': 'sam_hq_light'}]]


def record_model_builds(get_sam_model, get_grounding_dino_model, recorder):
    """Calls of both getters over MODEL_CONFIGS / GD_CONFIGS, with torch.load recording its path."""
    load = torch.load
    torch.load = lambda path: recorder.append(['torch.load', path]) or f'weights:{path}'
    try:
        out = []
        for c in MODEL_CONFIGS:
            recorder.clear()
            get_sam_model(c, 'cuda:0')
            out.append(list(recorder))
        for c in GD_CONFIGS:
            recorder.clear()
            get_grounding_dino_model(c, 'cuda:0')
            out.append(list(recorder))
        return out
    finally:
        torch.load = load


def segments_json(segments):
    """ObjectInfo list -> JSON-able [id, category_ids, isthing, scores]."""
    def plain(v):
        return None if v is None else (v.item() if hasattr(v, 'item') else v)
    return [[s.id, [plain(c) for c in s.category_ids], s.isthing, [plain(v) for v in s.scores]] for s in segments]
