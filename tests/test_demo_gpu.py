"""GPU: the demos' frames on the device - ``get_input_frame_for_deva``, ``DeviceLoader(SimpleVideoReader)``, CUDA frames
through the detectors and the result saver - against the fixtures minted from the unmodified reference, and the
reference's own processors run end to end over a demo clip with host frames and with device frames."""
import importlib.util
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'tracking-anything-with-deva_b200')
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
REF = os.path.join(ROOT, 'oracle', '_ref')


def _module(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(GOLDEN, f'{name}.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module')
def sc():
    sys.path.insert(0, GOLDEN)
    try:
        import demo_scenario
    finally:
        sys.path.remove(GOLDEN)
    return demo_scenario


@pytest.fixture(scope='module')
def golden():
    return json.load(open(os.path.join(GOLDEN, 'demo.json'))), dict(np.load(os.path.join(GOLDEN, 'demo.npz')))


def test_get_input_frame_matches_reference(sc, golden):
    """Within 1e-6 of the reference resized, bit for bit without a resize; numpy and CUDA input give the same bits."""
    from deva.inference.demo_utils import get_input_frame_for_deva
    meta, arrays = golden
    assert len(meta['ingest']) == len(sc.INGEST_SHAPES) * len(sc.INGEST_MIN_SIDES)
    for rec in meta['ingest']:
        k = int(rec['key'].split('_')[1])
        frame = sc.ingest_frame(*rec['hw'], k)
        a = get_input_frame_for_deva(frame, rec['min_side'])
        b = get_input_frame_for_deva(torch.from_numpy(frame).cuda(), rec['min_side'])
        assert a.is_cuda and a.dtype == torch.float32 and list(a.shape) == rec['shape'], rec
        assert torch.equal(a, b), rec
        ref = arrays[rec['key']]
        if rec['min_side'] <= 0:
            np.testing.assert_array_equal(a.cpu().numpy(), ref, err_msg=rec['key'])
        else:
            assert float(np.abs(a.cpu().numpy() - ref).max()) <= 1e-6, rec['key']


def _launches(monkeypatch):
    from deva.utils import jpeg_decode
    count, enqueue = [0], jpeg_decode.enqueue

    def counted(*a, **k):
        count[0] += 1
        return enqueue(*a, **k)
    monkeypatch.setattr(jpeg_decode, 'enqueue', counted)
    return count


def test_device_loader_reads_the_demo_clip(sc, golden, monkeypatch, tmp_path):
    from deva.inference.data.device_loader import DeviceLoader
    from deva.inference.data.simple_video_reader import SimpleVideoReader
    meta, _ = golden
    root = sc.write_demo_clip(str(tmp_path / 'clip'))
    reader = SimpleVideoReader(root)
    count = _launches(monkeypatch)
    loader = DeviceLoader(reader, prefetch=8)
    items = list(loader)
    assert count[0] == 3  # 12 frames in windows of 4: one JPEG launch per window
    assert loader.host_indices == sorted(sc.CLIP_SPECIAL)
    assert len(items) == len(reader) == len(meta['reader']['clip'])
    for i, ((frame, p), want) in enumerate(zip(items, meta['reader']['clip'])):
        assert frame.is_cuda and frame.dtype == torch.uint8 and p == reader[i][1]
        assert torch.equal(frame.cpu(), torch.from_numpy(reader[i][0])), i
        assert [os.path.relpath(p, root), sc.sha(frame.cpu().numpy()), list(frame.shape)] == want


def test_device_loader_reads_mixed_files_like_the_reader(sc, golden, monkeypatch, tmp_path):
    """Declined files (progressive, grayscale, CMYK, PNG) are the reader's items; a file Pillow cannot read raises the
    reader's error at its index."""
    from deva.inference.data.device_loader import DeviceLoader
    from deva.inference.data.simple_video_reader import SimpleVideoReader
    meta, _ = golden
    root = sc.write_reader_folder(str(tmp_path / 'reader'))
    reader = SimpleVideoReader(root)
    count = _launches(monkeypatch)
    loader = DeviceLoader(reader, prefetch=4)
    got = []
    with pytest.raises(Exception) as err:
        for frame, p in loader:
            got.append([os.path.relpath(p, root), sc.sha(frame.cpu().numpy()), list(frame.shape)])
    want = meta['reader']['reader']
    bad = [i for i, w in enumerate(want) if len(w[1]) != 64][0]
    assert got == want[:bad]
    assert [type(err.value).__name__, str(err.value).replace(root, '<root>')] == want[bad][1:]
    assert loader.host_indices == [2, 3, 4, 5, 6, bad]
    # windows of 2: files 0-1 and file 8 are the device's JPEGs; file 8's window is enqueued before file 7 is handed out
    assert count[0] == 2


def _cuda_image_saver(ResultSaver):
    class CudaImageSaver(ResultSaver):
        def save_mask(self, *args, image_np=None, **kwargs):
            if image_np is not None:
                image_np = torch.from_numpy(image_np).cuda()
            super().save_mask(*args, image_np=image_np, **kwargs)
    return CudaImageSaver


@pytest.mark.parametrize('index', range(8))
def test_saver_replay_with_cuda_images(index):
    """The saver sessions with every image_np handed over as a CUDA tensor write what the reference wrote."""
    ss = _module('saver_session')
    meta = json.load(open(os.path.join(GOLDEN, 'saver.json')))
    arrays = np.load(os.path.join(GOLDEN, 'saver.npz'))
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    expected = meta['sessions'][index]
    rec = ss.Recorder()
    with rec.installed() as orig_save, tempfile.TemporaryDirectory() as root:
        video_json = ss.drive(_cuda_image_saver(ResultSaver), ObjectManager, ObjectInfo, ss.SESSIONS[index],
                              expected['seeds'], root, rec, orig_save, to_prob=lambda p: p.cuda())
    assert json.loads(json.dumps(video_json)) == expected['video_json']
    assert len(rec.events) == len(expected['events'])
    for got, want in zip(rec.events, expected['events']):
        if isinstance(got[-1], np.ndarray):
            assert list(got[:-1]) == want[:-1]
            assert np.array_equal(got[-1], arrays[want[-1]]), want
        else:
            assert json.loads(json.dumps(list(got))) == want


def test_saver_downloads_a_cuda_image_of_another_shape():
    """A CUDA image_np that is not uint8 [h, w, 3] of the output size is blended as the numpy array it holds."""
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    from PIL import Image
    prob = torch.rand(3, 24, 32, device='cuda')
    image = np.random.default_rng(3).integers(0, 256, (24, 32, 3)).astype(np.float32)
    out = {}
    with tempfile.TemporaryDirectory() as root:
        for name, img in (('np', image), ('cuda', torch.from_numpy(image).cuda())):
            om = ObjectManager()
            om.use_long_id = True
            om.add_new_objects([ObjectInfo(300), ObjectInfo(70000)])
            saver = ResultSaver(os.path.join(root, name), None, dataset='demo', object_manager=om)
            saver.save_mask(prob, '00000.jpg', image_np=img)
            saver.end()
            out[name] = np.array(Image.open(os.path.join(root, name, 'Visualizations', '00000.jpg')))
    assert np.array_equal(out['np'], out['cuda'])


def test_detectors_with_cuda_images_match_reference():
    """auto_segment and segment_with_text given the images as CUDA tensors reproduce detector_masks.{json,npz}, the
    fakes' recorded calls included."""
    from deva.ext.automatic_sam import auto_segment
    from deva.ext.grounding_dino import segment_with_text
    dms = _module('detector_masks_scenario')
    meta = json.load(open(os.path.join(GOLDEN, 'detector_masks.json')))
    arrays = dict(np.load(os.path.join(GOLDEN, 'detector_masks.npz')))
    for case, rec in zip(dms.AUTO_CASES, meta['auto']):
        name, (h, w), min_side, suppress, thr, fwd, spec = case
        masks = dms.build_masks(spec, h, w, rec['seed'])
        sam = dms.FakeAutoSam(masks, dms.iou_preds(len(masks), rec['seed']), 'cuda')
        fm = dms.forward_mask(fwd, h, w)
        out, segs = auto_segment(dms.auto_config(thr), sam, torch.from_numpy(dms.image(h, w)).cuda(),
                                 None if fm is None else fm.cuda(), min_side, suppress)
        np.testing.assert_array_equal(out.cpu().numpy(), arrays[f'auto_{name}'], err_msg=name)
        assert dms.segments_json(segs) == rec['segments'], name
        assert [c[:3] for c in sam.calls] == [c[:3] for c in rec['calls']], name
        for got, want in zip(sam.calls, rec['calls']):
            assert len(got[3]) == len(want[3]), name
            for a, b in zip(got[3], want[3]):
                assert (a is None and b is None) or np.allclose(a, b, rtol=0, atol=1e-6), name
    for case, rec in zip(dms.TEXT_CASES, meta['text']):
        name, (h, w), min_side, nms, boxes = case
        gd, sam = dms.FakeGroundingDino(boxes, 'cuda'), dms.FakeSamPredictor()
        out, segs = segment_with_text(dms.text_config(nms), gd, sam, torch.from_numpy(dms.image(h, w)).cuda(),
                                      ['a', 'b'], min_side)
        np.testing.assert_array_equal(out.cpu().numpy(), arrays[f'text_{name}'], err_msg=name)
        assert dms.segments_json(segs) == rec['segments'], name
        assert json.loads(json.dumps(gd.calls + sam.calls)) == rec['calls'], name


# the reference's processors over the demo clip, run in a subprocess with this package first on the path and the
# staged reference after it; prints one JSON object per (run, encoders, arm)
DEMO_LOOP = r'''
import hashlib, json, os, sys, tempfile, types
sys.path.insert(0, GOLDEN)
import numpy as np, torch
from torch.utils.data import DataLoader
import demo_scenario as sc, detector_masks_scenario as dms

dms.install_detector_stubs([])
sv = sys.modules['supervision'] = types.ModuleType('supervision')  # boxes painted, labels ignored: deterministic


class Detections:
    def __init__(self, xyxy, confidence=None, class_id=None):
        self.xyxy = xyxy


class BoundingBoxAnnotator:
    def annotate(self, scene, detections):
        scene = scene.copy()
        for x0, y0, x1, y1 in detections.xyxy.astype(int):
            scene[y0:y1 + 1, x0:x1 + 1][[0, -1]] = 255
        return scene


class LabelAnnotator:
    def annotate(self, scene, detections, labels=None):
        return scene.copy()


sv.Detections, sv.BoundingBoxAnnotator, sv.LabelAnnotator = Detections, BoundingBoxAnnotator, LabelAnnotator
from deva.ext import automatic_processor, with_text_processor
assert automatic_processor.__file__.startswith(REF) and with_text_processor.__file__.startswith(REF)
from deva.inference.data.device_loader import DeviceLoader
from deva.inference.data.simple_video_reader import SimpleVideoReader, no_collate
from deva.inference.demo_utils import flush_buffer
from deva.inference.inference_core import DEVAInferenceCore
from deva.inference.result_utils import ResultSaver
from deva.model.network import DEVA
from deva.model.param_spec import synthetic_state_dict

CFG = dict(key_dim=64, value_dim=512, pix_feat_dim=512, mem_every=5, enable_long_term=True, chunk_size=-1, top_k=30,
           enable_long_term_count_usage=False, max_mid_term_frames=10, min_mid_term_frames=5, num_prototypes=128,
           max_long_term_elements=10000)
sd = {k: v.cuda() for k, v in synthetic_state_dict(seed=1).items()}
saves = []


class Recording(ResultSaver):
    def save_mask(self, *args, **kwargs):
        rec = sc.SaveRecorder(lambda im: im.cpu().numpy() if torch.is_tensor(im) else im)
        rec.save_mask(*args, **kwargs)
        saves.append(rec.calls[0])
        super().save_mask(*args, **kwargs)


torch.autograd.set_grad_enabled(False)
with tempfile.TemporaryDirectory() as tmp:
    clip = sc.write_demo_clip(os.path.join(tmp, 'clip'))
    for kind, temporal in sc.RUNS:
        for enc in ('pil', 'device'):
            for arm in ('A', 'B'):
                np.random.seed(42)
                cfg = sc.demo_config(CFG, kind, temporal)
                net = DEVA(cfg).cuda().eval()
                net.load_weights(sd)
                deva = DEVAInferenceCore(net, config=cfg)
                out = os.path.join(tmp, f'{kind}_{temporal}_{enc}_{arm}')
                saves.clear()
                saver = Recording(out, None, dataset='demo', object_manager=deva.object_manager, png_encoder=enc,
                                  jpeg_encoder=enc)
                reader = SimpleVideoReader(clip)
                frames = DataLoader(reader, batch_size=None, collate_fn=no_collate, num_workers=0) if arm == 'A' \
                    else DeviceLoader(reader)
                args, fakes = sc.detectors(kind, 'cuda')
                processors = automatic_processor if kind == 'auto' else with_text_processor
                sc.run_demo(processors, flush_buffer, deva, frames, kind, saver, args)
                saver.end()
                with open(os.path.join(out, 'pred.json'), 'w') as f:
                    json.dump(saver.video_json, f, indent=4)
                files = {}
                for d, _, names in os.walk(out):
                    for n in names:
                        p = os.path.join(d, n)
                        files[os.path.relpath(p, out)] = hashlib.sha256(open(p, 'rb').read()).hexdigest()
                print(json.dumps({'kind': kind, 'temporal': temporal, 'enc': enc, 'arm': arm, 'files': files,
                                  'calls': sc.calls(fakes), 'calls_no_points': sc.calls(fakes, False),
                                  'saves': list(saves),
                                  'host_indices': getattr(frames, 'host_indices', None)}))
'''


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, 'deva', 'ext', 'automatic_processor.py')),
                    reason='oracle/_ref not staged (python oracle/build_ref.py && python oracle/build_ref_demo.py)')
def test_reference_demo_loop_with_device_frames(sc, golden):
    """Arm A (the demo's DataLoader, numpy frames) and arm B (DeviceLoader, CUDA frames) write byte-identical files and
    pred.json and make identical detector calls, point prompts included; both match the reference's call sequence."""
    meta, _ = golden
    code = f'GOLDEN, REF = {GOLDEN!r}, {REF!r}\n' + DEMO_LOOP
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, REF, ROOT]))
    out = subprocess.run([sys.executable, '-c', code], env=env, capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-4000:]
    results = [json.loads(line) for line in out.stdout.splitlines() if line.startswith('{')]
    assert len(results) == len(sc.RUNS) * 4
    want = {(r['kind'], r['temporal']): r for r in meta['runs']}
    for a, b in zip(results[0::2], results[1::2]):
        tag = (a['kind'], a['temporal'], a['enc'])
        assert (a['arm'], b['arm']) == ('A', 'B') and b['host_indices'] == sorted(sc.CLIP_SPECIAL), tag
        assert len(a['files']) == 2 * sc.CLIP_FRAMES + 1 and a['files'] == b['files'], tag
        assert a['calls'] == b['calls'] and a['saves'] == b['saves'], tag
        ref = want[(a['kind'], a['temporal'])]
        assert a['calls_no_points'] == ref['detector_calls'], tag
        assert a['saves'] == ref['saves'], tag
