"""PNG files encoded on the device (csrc/png.cu, deva/utils/png_encode.py): byte for byte oracle/png_encode.py's files
over the CPU test's matrix, deterministic, and a drop-in for Pillow's files in the result saver (the
tests/golden/saver.{json,npz} replay), limit_max_id (tests/golden/unsup_davis17.*) and merge_stuff
(tests/golden/vps_metrics.*): every PNG decodes to the recorded pixels, mode and palette, and everything else the
passes write is unchanged.  save_mask with the device encoder still never synchronises the host."""
import functools
import hashlib
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
import png_cases as pc  # noqa: E402

from oracle import png_encode as op  # noqa: E402

pytestmark = pytest.mark.gpu


def _device(case):
    img, mode, palette = pc.make(case)
    return torch.from_numpy(img).cuda(), img, mode, palette


@pytest.mark.parametrize('case', pc.case_ids(large=False) + pc.case_ids(large=True))
def test_device_matches_oracle(case):
    from deva.utils.png_encode import encode_png
    dev, img, mode, palette = _device(case)
    got = encode_png(dev, mode, palette)
    want = op.encode_png(img, mode, palette)
    assert got == want, (case, len(got), len(want))


def test_encodes_are_deterministic():
    """Two encodes of one image, and several in flight at once on one stream, give identical bytes."""
    from deva.utils.png_encode import encode_png, encode_png_async
    dev, _, mode, palette = _device('RGB-ellipse-1080x1920')
    first = encode_png(dev, mode, palette)
    assert encode_png(dev, mode, palette) == first
    pending = [encode_png_async(dev, mode, palette) for _ in range(4)]
    assert all(p.result() == first for p in pending)


def test_unaligned_and_strided_inputs():
    """A view at an odd offset and a non-contiguous view encode like their contiguous copies."""
    from deva.utils.png_encode import encode_png
    _, img, _, _ = _device('L-ellipse-37x53')
    buf = torch.zeros(img.size + 1, dtype=torch.uint8, device='cuda')
    buf[1:] = torch.from_numpy(img.reshape(-1)).cuda()
    assert encode_png(buf[1:].view(img.shape), 'L') == op.encode_png(img, 'L')
    wide = torch.from_numpy(np.ascontiguousarray(np.tile(img, (1, 2)))).cuda()
    assert encode_png(wide[:, ::2], 'L') == op.encode_png(np.tile(img, (1, 2))[:, ::2], 'L')


def test_rejects_bad_images():
    from deva.utils.png_encode import encode_png
    with pytest.raises(ValueError, match='RGB'):
        encode_png(torch.zeros(4, 5, dtype=torch.uint8, device='cuda'), 'RGB')
    with pytest.raises(ValueError, match='uint8'):
        encode_png(torch.zeros(4, 5, dtype=torch.int32, device='cuda'), 'L')


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


def _is_png_event(e):
    return e[0] == 'image' and e[1].endswith('.png')


@pytest.mark.parametrize('index', range(8))
def test_saver_replay_with_device_png(saver_fixture, index):
    """The saver fixture with png_encoder='device': the JSON and every non-PNG event as recorded; every PNG file
    decodes to the recorded mode, palette and pixels, and no other PNG is written."""
    ss, meta, arrays = saver_fixture
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    expected = meta['sessions'][index]
    rec = ss.Recorder()
    with rec.installed() as orig_save, tempfile.TemporaryDirectory() as root:
        video_json = ss.drive(functools.partial(ResultSaver, png_encoder='device'), ObjectManager, ObjectInfo,
                              ss.SESSIONS[index], expected['seeds'], root, rec, orig_save, to_prob=lambda p: p.cuda())
        written = sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs
                         if f.endswith('.png') and not f.startswith('input_'))
        pngs = [e for e in expected['events'] if _is_png_event(e)]
        assert written == sorted(e[1] for e in pngs)
        for _, rel, mode, pal, key in pngs:
            img = Image.open(os.path.join(root, rel))
            assert img.mode == mode, rel
            assert (img.getpalette() if img.mode == 'P' else None) == pal, rel
            np.testing.assert_array_equal(np.asarray(img), arrays[key])
    assert json.loads(json.dumps(video_json)) == expected['video_json']
    rest = [e for e in expected['events'] if not _is_png_event(e)]
    assert len(rec.events) == len(rest)
    for got, want in zip(rec.events, rest):
        if isinstance(got[-1], np.ndarray):
            assert list(got[:-1]) == want[:-1], (got[:-1], want[:-1])
            assert np.array_equal(got[-1], arrays[want[-1]]), want
        else:
            assert json.loads(json.dumps(list(got))) == want


def test_save_mask_with_device_png_does_not_synchronise(saver_fixture):
    """The device path (uint8 frame, overlay, prompts, JSON, device PNG) enqueues its work without a host
    synchronisation, also for a stream longer than the prefix copied with the encode."""
    ss = saver_fixture[0]
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    om = ObjectManager()
    om.use_long_id = True
    om.add_new_objects([ObjectInfo(300, category_id=0, score=0.9), ObjectInfo(70000, category_id=1, score=0.5)])
    rec = ss.Recorder()
    with rec.installed(), tempfile.TemporaryDirectory() as root:
        saver = ResultSaver(root, None, dataset='demo', object_manager=om, png_encoder='device')
        prob = torch.from_numpy(ss.make_prob(5, 3)).cuda()
        g = torch.Generator('cuda').manual_seed(0)
        noisy = torch.softmax(20 * torch.randn(3, 1024, 1024, device='cuda', generator=g), 0)  # a noisy id map
        noisy_image = np.zeros((1024, 1024, 3), np.uint8)
        image = ss.make_image(5, ss.OUT)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            for t in range(3):
                saver.save_mask(prob, f'{t:05d}.jpg', need_resize=True, shape=ss.OUT, image_np=image,
                                prompts=ss.PROMPTS)
            saver.save_mask(noisy, '00003.jpg', image_np=noisy_image)
        finally:
            torch.cuda.set_sync_debug_mode('default')
        saver.end()
        files = sorted(os.listdir(os.path.join(root, 'Annotations')))
        assert files == [f'{t:05d}.png' for t in range(4)]
        big = os.path.getsize(os.path.join(root, 'Annotations', '00003.png'))
        from deva.utils.png_encode import PREFIX
        assert big > PREFIX
        assert Image.open(os.path.join(root, 'Annotations', '00003.png')).size == (1024, 1024)
    assert [e[0] for e in rec.events].count('image') == 4  # the overlays; the PNGs do not go through Pillow


# ---------------------------------------------------------------------------------------------- post-processing
def test_limit_max_id_with_device_png_matches_reference(tmp_path):
    import unsup_davis_scenario as us
    from deva.inference.postprocess_unsup_davis17 import limit_max_id
    meta = json.load(open(os.path.join(GOLDEN, 'unsup_davis17.json')))
    arrays = np.load(os.path.join(GOLDEN, 'unsup_davis17.npz'))
    palette = bytes.fromhex(meta['palette'])
    for case in us.CASES:
        root = tmp_path / case
        root.mkdir()
        error, files = us.run_case(
            lambda src, dst, m: limit_max_id(src, dst, m, palette=palette, png_encoder='device'), str(root), case)
        us.assert_matches(meta, arrays, case, error, files)


def test_merge_stuff_with_device_png_matches_reference(tmp_path):
    import vps_scenario as vs
    from deva.vps_metrics.stuff_merging import merge_stuff
    from deva.vps_metrics.video_pass import read_rgb
    meta = json.load(open(os.path.join(GOLDEN, 'vps_metrics.json')))
    arrays = np.load(os.path.join(GOLDEN, 'vps_metrics.npz'))
    (tmp_path / 'data').mkdir()
    dataset = vs.write_dataset(str(tmp_path / 'data'))
    out = str(tmp_path / 'merged')
    np.random.seed(meta['merge_seed'])
    merge_stuff(dataset[0], out, isthing={int(k): v for k, v in meta['isthing'].items()}, png_encoder='device')
    assert json.load(open(os.path.join(out, 'pred.json'))) == meta['merged_json']
    for key, digest in meta['merged_sha256'].items():
        assert Image.open(os.path.join(out, 'pan_pred', key)).mode == 'RGB'
        assert hashlib.sha256(read_rgb(os.path.join(out, 'pan_pred', key)).tobytes()).hexdigest() == digest, key
    for key in arrays.files:
        if key.startswith('merged_'):
            vid, t = key[len('merged_'):].rsplit('_', 1)
            np.testing.assert_array_equal(read_rgb(os.path.join(out, 'pan_pred', vid, f'{int(t):08d}.png')),
                                          arrays[key])
