"""CPU: the detector-mask oracle against the fixture minted from the reference, the CPU bilinear threshold decisions it
restates, and the drop-in modules' imports and model builds (no detector package, no GPU)."""
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F
import torchvision

from oracle import detector_masks as om

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'tracking-anything-with-deva_b200')
REFERENCE = os.environ.get('DEVA_REFERENCE_ROOT', '/root/reference')


@pytest.fixture(scope='module')
def sc(golden_dir):
    spec = importlib.util.spec_from_file_location('detector_masks_scenario',
                                                  os.path.join(golden_dir, 'detector_masks_scenario.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module')
def golden(golden_dir):
    meta = json.load(open(os.path.join(golden_dir, 'detector_masks.json')))
    return meta, dict(np.load(os.path.join(golden_dir, 'detector_masks.npz')))


def _size(h, w, min_side):
    return (int(h * min_side / min(h, w)), int(w * min_side / min(h, w))) if min_side > 0 else (h, w)


def text_detections(sc, case):
    """The text path up to the mask stack, as the reference makes it: detector, CPU NMS, best of three SAM masks."""
    name, (h, w), min_side, nms, boxes = case
    gd, sam = sc.FakeGroundingDino(boxes, 'cpu'), sc.FakeSamPredictor()
    img = sc.image(h, w)
    sam.set_image(img)
    det = gd.predict_with_classes(img[..., ::-1], ['a', 'b'], 0.35, 0.35)
    keep = torchvision.ops.nms(torch.from_numpy(det.xyxy), torch.from_numpy(det.confidence), nms).numpy().tolist()
    masks = []
    for box in det.xyxy[keep]:
        m, s, _ = sam.predict(box=box, multimask_output=True)
        masks.append(m[np.argmax(s)])
    return np.array(masks), det.confidence[keep], det.class_id[keep]


def test_oracle_reproduces_auto_cases(sc, golden):
    meta, arrays = golden
    assert [c['name'] for c in meta['auto']] == [c[0] for c in sc.AUTO_CASES]
    for case, rec in zip(sc.AUTO_CASES, meta['auto']):
        name, (h, w), min_side, suppress, thr, fwd, spec = case
        out_h, out_w = _size(h, w, min_side)
        if fwd == 'all':  # no positive point: the reference returns before generating
            assert rec['calls'] == [] and not arrays[f'auto_{name}'].any() and rec['segments'] == []
            continue
        masks = sc.build_masks(spec, h, w, rec['seed'])
        out, segs = om.scored_id_map(masks, sc.iou_preds(len(masks), rec['seed']), out_h, out_w, suppress, thr)
        np.testing.assert_array_equal(out, arrays[f'auto_{name}'], err_msg=name)
        assert [[i, [None], None, [s]] for i, s in segs] == rec['segments'], name


def test_oracle_reproduces_text_cases(sc, golden):
    meta, arrays = golden
    assert [c['name'] for c in meta['text']] == [c[0] for c in sc.TEXT_CASES]
    for case, rec in zip(sc.TEXT_CASES, meta['text']):
        masks, conf, cls = text_detections(sc, case)
        out, segs = om.cover_id_map(masks, *_size(*case[1], case[2]))
        np.testing.assert_array_equal(out, arrays[f'text_{case[0]}'], err_msg=case[0])
        expect = sc.segments_json([type('S', (), dict(id=i, category_ids=[cls[k]], isthing=None,
                                                      scores=[conf[k]]))() for i, k in segs])
        assert expect == rec['segments'], case[0]


def test_fixture_is_self_consistent(sc, golden):
    meta, arrays = golden
    free = {c[0] for c in sc.AUTO_CASES if not c[3]}  # without suppress_small_mask the map holds channels, not ids
    for rec in meta['auto'] + meta['text']:
        kind = 'auto' if rec in meta['auto'] else 'text'
        m = arrays[f'{kind}_{rec["name"]}']
        ids = [s[0] for s in rec['segments']]
        assert ids == list(range(1, len(ids) + 1)), rec['name']
        if kind == 'text' or rec['name'] not in free:  # painted maps hold listed ids only (an id may be overwritten)
            assert set(np.unique(m).tolist()) <= {0, *ids}, rec['name']
    by_name = {r['name']: r for r in meta['auto']}
    # planted semantics: the float32 boundary mask is accepted; the free path's ids and channels disagree
    assert len(by_name['f32_boundary']['segments']) == 2
    mismatch = arrays['auto_free_id_channel_mismatch']
    assert set(np.unique(mismatch).tolist()) == {0, 2, 4} and len(by_name['free_id_channel_mismatch']['segments']) == 2
    assert by_name['forward_points']['calls'][0][3][0] is not None  # positive points were passed
    text = {r['name']: r for r in meta['text']}
    assert text['no_boxes']['segments'] == [] and not arrays['text_no_boxes'].any()
    assert len(text['empty_after_resize']['segments']) == 3  # 4 boxes, one vanishes at 60 px
    assert [s[1] for s in text['none_class_ids']['segments']].count([None]) >= 1
    assert sum(c[0] == 'predict' for c in text['nms_suppression']['calls']) == 2


def test_oracle_threshold_decisions_equal_torch_cpu_bilinear():
    """v > 0.5 and v >= 0.5 of the restated (kernel) arithmetic equal F.interpolate's on the CPU, which the reference's
    segment_with_text thresholds: random masks over a few hundred random scales, and the demo's 1080p / 720p shapes."""
    rng = np.random.default_rng(0)
    shapes = [(int(rng.integers(1, 160)), int(rng.integers(1, 160)), int(rng.integers(1, 200)), int(rng.integers(1, 200)))
              for _ in range(300)]
    shapes += [(1080, 1920, 480, 853), (720, 1280, 480, 853), (333, 517, 480, 745), (96, 128, 48, 64), (48, 64, 96, 128)]
    for h, w, oh, ow in shapes:
        m = rng.random((2, h, w)) < rng.uniform(0.05, 0.95)
        if h > 8 and w > 8:  # plus blocky masks: long runs of equal values
            m[1] = np.kron(rng.random((h // 8 + 1, w // 8 + 1)) < 0.5, np.ones((8, 8), bool))[:h, :w]
        t = F.interpolate(torch.from_numpy(m).float()[None], (oh, ow), mode='bilinear')[0].numpy()
        o = om.resize(m, oh, ow)
        assert ((t > 0.5) == (o > 0.5)).all() and ((t >= 0.5) == (o >= 0.5)).all(), (h, w, oh, ow)


def _run(code, *paths):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(paths))
    out = subprocess.run([sys.executable, '-c', code], env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


def test_ext_modules_import_without_detectors_and_cuda():
    _run("import sys\n"
         "for m in ('segment_anything', 'groundingdino', 'GroundingDINO', 'supervision'):\n"
         "    sys.modules[m] = None\n"
         "import torch\n"
         "import deva.ext.automatic_sam as a, deva.ext.grounding_dino as g\n"
         f"assert a.__file__.startswith({PKG!r}) and g.__file__.startswith({PKG!r})\n"
         "assert callable(a.auto_segment) and callable(g.segment_with_text)\n"
         "assert not torch.cuda.is_initialized()\n", PKG)


def test_model_getters_make_the_recorded_calls(sc, golden):
    meta, _ = golden
    saved = dict(sys.modules)
    try:
        recorder = []
        sc.install_detector_stubs(recorder)
        from deva.ext.automatic_sam import get_sam_model
        from deva.ext.grounding_dino import get_grounding_dino_model
        got = sc.record_model_builds(get_sam_model, get_grounding_dino_model, recorder)
    finally:
        for k in set(sys.modules) - set(saved):
            del sys.modules[k]
        sys.modules.update(saved)
    assert json.loads(json.dumps(got)) == meta['model_builds']


@pytest.mark.skipif(not os.path.isdir(os.path.join(REFERENCE, 'deva', 'ext')), reason='no reference checkout')
def test_reference_processors_resolve_to_this_package():
    """With this package first on sys.path, the reference's processors take auto_segment / segment_with_text from here,
    and the rest of deva.ext (ext_eval_args, SAM) still resolves to the checkout."""
    _run("import sys, types\n"
         "for name in ('segment_anything', 'groundingdino', 'groundingdino.util', 'groundingdino.util.inference'):\n"
         "    m = sys.modules[name] = types.ModuleType(name); m.__path__ = []\n"
         "    m.SamAutomaticMaskGenerator = m.SamPredictor = m.Model = object\n"
         "sys.modules['pulp'] = types.ModuleType('pulp')\n"
         "import deva.ext.automatic_processor as ap, deva.ext.with_text_processor as tp, deva.ext.ext_eval_args as ea\n"
         f"assert ap.auto_segment.__module__ == 'deva.ext.automatic_sam' and ap.auto_segment.__code__.co_filename.startswith({PKG!r})\n"
         f"assert tp.segment_with_text.__code__.co_filename.startswith({PKG!r})\n"
         f"assert ea.__file__.startswith({REFERENCE!r}) and ap.__file__.startswith({REFERENCE!r})\n", PKG, REFERENCE)
