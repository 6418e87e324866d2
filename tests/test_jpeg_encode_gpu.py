"""Baseline JPEG files encoded on the device (csrc/jpeg.cu, deva/utils/jpeg_encode.py): byte for byte
oracle/jpeg_encode.py's files over the CPU test's matrix and Pillow's own at 1080p and 4K, deterministic, the same from
numpy and CUDA input, and enqueued without a host synchronisation.  In the result saver (the
tests/golden/saver.{json,npz} replay) with jpeg_encoder='device', alone and with png_encoder='device', every overlay
JPEG is Pillow's encode of the recorded image and every other output is unchanged."""
import functools
import io
import json
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
from PIL import Image

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
sys.path.insert(0, GOLDEN)
import jpeg_cases as jc  # noqa: E402

from oracle import jpeg_encode as oj  # noqa: E402

pytestmark = pytest.mark.gpu


def _pillow(img, quality=75):
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, 'JPEG', quality=quality)
    return buf.getvalue()


@pytest.mark.parametrize('case', jc.case_ids(large=False) + jc.case_ids(large=True))
def test_device_matches_oracle(case):
    from deva.utils.jpeg_encode import encode_jpeg
    img, q = jc.make(case)
    got = encode_jpeg(torch.from_numpy(img).cuda(), q)
    want = oj.encode_jpeg(img, q)
    assert got == want, (case, len(got), len(want))


@pytest.mark.parametrize('shape', [(1080, 1920), (2160, 3840)])
@pytest.mark.parametrize('k', [16, 50])
def test_device_matches_pillow_at_1080p_and_4k(shape, k):
    from deva.utils.jpeg_encode import encode_jpeg
    img = jc.overlay(*shape, k=k)
    assert encode_jpeg(torch.from_numpy(img).cuda()) == _pillow(img)


def test_noise_4k_matches_pillow():
    """A scan far longer than the prefix copied with the encode, with thousands of stuffed bytes."""
    from deva.utils.jpeg_encode import PREFIX, encode_jpeg
    img = np.random.default_rng(4).integers(0, 256, (2160, 3840, 3), dtype=np.uint8)
    data = encode_jpeg(img, 95)
    assert len(data) > 4 * PREFIX
    assert data == _pillow(img, 95)


def test_encodes_are_deterministic():
    """Two encodes of one image, and several in flight at once on one stream, give identical bytes."""
    from deva.utils.jpeg_encode import encode_jpeg, encode_jpeg_async
    dev = torch.from_numpy(jc.overlay(1080, 1920, k=50)).cuda()
    first = encode_jpeg(dev)
    assert encode_jpeg(dev) == first
    pending = [encode_jpeg_async(dev) for _ in range(4)]
    assert all(p.result() == first for p in pending)


def test_numpy_and_cuda_inputs_agree():
    from deva.utils.jpeg_encode import encode_jpeg
    img, q = jc.make('overlay-481x857-q75')
    assert encode_jpeg(img, q) == encode_jpeg(torch.from_numpy(img).cuda(), q) == oj.encode_jpeg(img, q)
    wide = torch.from_numpy(np.ascontiguousarray(np.tile(img, (1, 2, 1)))).cuda()
    assert encode_jpeg(wide[:, ::2]) == oj.encode_jpeg(np.tile(img, (1, 2, 1))[:, ::2])  # a strided view


def test_encode_async_does_not_synchronise():
    from deva.utils.jpeg_encode import encode_jpeg_async
    dev = torch.from_numpy(jc.overlay(1080, 1920)).cuda()
    encode_jpeg_async(dev).result()  # warm the allocator and the library
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        pending = [encode_jpeg_async(dev, quality=q) for q in (75, 90)]
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert pending[0].result() == _pillow(jc.overlay(1080, 1920))


def test_rejects_bad_images():
    from deva.utils.jpeg_encode import encode_jpeg
    for bad in (torch.zeros(4, 5, dtype=torch.uint8, device='cuda'), torch.zeros(4, 5, 4, dtype=torch.uint8,
                                                                                device='cuda'),
                torch.zeros(4, 5, 3, dtype=torch.int32, device='cuda'), torch.zeros(4, 5, 3, dtype=torch.uint8),
                torch.zeros(1, 65536, 3, dtype=torch.uint8, device='cuda')):
        with pytest.raises(ValueError):
            encode_jpeg(bad)
    with pytest.raises(ValueError, match='quality'):
        encode_jpeg(torch.zeros(4, 5, 3, dtype=torch.uint8, device='cuda'), quality=0)


# ---------------------------------------------------------------------------------------------- result saver
def _session_module():
    import importlib.util
    spec = importlib.util.spec_from_file_location('saver_session', os.path.join(GOLDEN, 'saver_session.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module')
def saver_fixture():
    meta = json.load(open(os.path.join(GOLDEN, 'saver.json')))
    return _session_module(), meta, np.load(os.path.join(GOLDEN, 'saver.npz'))


def _is_jpg_event(e):
    return e[0] == 'image' and e[1].endswith('.jpg')


def _is_png_event(e):
    return e[0] == 'image' and e[1].endswith('.png')


@pytest.mark.parametrize('png_encoder', ['pil', 'device'])
@pytest.mark.parametrize('index', range(8))
def test_saver_replay_with_device_jpeg(saver_fixture, index, png_encoder):
    """The saver fixture with jpeg_encoder='device': every overlay JPEG is byte for byte Pillow's encode of the
    recorded image (the prompt and host-blend frames included) and no other JPEG is written; the JSON and every other
    event as recorded (PNGs decode to the recorded pixels when they are encoded on the device too)."""
    ss, meta, arrays = saver_fixture
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    expected = meta['sessions'][index]
    rec = ss.Recorder()
    with rec.installed() as orig_save, tempfile.TemporaryDirectory() as root:
        saver = functools.partial(ResultSaver, jpeg_encoder='device', png_encoder=png_encoder)
        video_json = ss.drive(saver, ObjectManager, ObjectInfo, ss.SESSIONS[index], expected['seeds'], root, rec,
                              orig_save, to_prob=lambda p: p.cuda())
        on_disk = lambda ext: sorted(os.path.relpath(os.path.join(d, f), root)  # noqa: E731
                                     for d, _, fs in os.walk(root) for f in fs
                                     if f.endswith(ext) and not f.startswith('input_'))
        jpgs = [e for e in expected['events'] if _is_jpg_event(e)]
        assert on_disk('.jpg') == sorted(e[1] for e in jpgs)
        for _, rel, mode, _, key in jpgs:
            assert mode == 'RGB'
            buf = io.BytesIO()
            orig_save(Image.fromarray(arrays[key]), buf, 'JPEG')
            assert open(os.path.join(root, rel), 'rb').read() == buf.getvalue(), rel
        pngs = [e for e in expected['events'] if _is_png_event(e)]
        if png_encoder == 'device':
            assert on_disk('.png') == sorted(e[1] for e in pngs)
            for _, rel, mode, pal, key in pngs:
                img = Image.open(os.path.join(root, rel))
                assert img.mode == mode and (img.getpalette() if img.mode == 'P' else None) == pal, rel
                np.testing.assert_array_equal(np.asarray(img), arrays[key])
    assert json.loads(json.dumps(video_json)) == expected['video_json']
    skip = _is_jpg_event if png_encoder == 'pil' else (lambda e: _is_jpg_event(e) or _is_png_event(e))
    rest = [e for e in expected['events'] if not skip(e)]
    assert len(rec.events) == len(rest)
    for got, want in zip(rec.events, rest):
        if isinstance(got[-1], np.ndarray):
            assert list(got[:-1]) == want[:-1], (got[:-1], want[:-1])
            assert np.array_equal(got[-1], arrays[want[-1]]), want
        else:
            assert json.loads(json.dumps(list(got))) == want


def test_save_mask_with_device_jpeg_does_not_synchronise(saver_fixture):
    """The device overlay path (uint8 frame, no prompts, device PNG and JPEG) enqueues its work without a host
    synchronisation; the files are Pillow's JPEGs of the blend the pil path writes."""
    ss = saver_fixture[0]
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    om = ObjectManager()
    om.use_long_id = True
    om.add_new_objects([ObjectInfo(300, category_id=0, score=0.9), ObjectInfo(70000, category_id=1, score=0.5)])
    prob = torch.from_numpy(ss.make_prob(5, 3)).cuda()
    image = jc.frame(*ss.OUT)
    outputs = {}
    for enc in ('pil', 'device'):
        with tempfile.TemporaryDirectory() as root:
            saver = ResultSaver(root, None, dataset='demo', object_manager=om, png_encoder=enc, jpeg_encoder=enc)
            saver.save_mask(prob, '00000.jpg', need_resize=True, shape=ss.OUT, image_np=image)  # warm up
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode('error' if enc == 'device' else 'default')
            try:
                for t in range(1, 4):
                    saver.save_mask(prob, f'{t:05d}.jpg', need_resize=True, shape=ss.OUT, image_np=image)
            finally:
                torch.cuda.set_sync_debug_mode('default')
            saver.end()
            outputs[enc] = {f: open(os.path.join(root, 'Visualizations', f), 'rb').read()
                            for f in sorted(os.listdir(os.path.join(root, 'Visualizations')))}
    assert list(outputs['device']) == [f'{t:05d}.jpg' for t in range(4)]
    assert outputs['device'] == outputs['pil']
