"""ResultSaver with ``jpeg_decoder='device'`` against the same saver with ``jpeg_decoder='pil'``: the saver sessions of
tests/golden/saver_session.py replayed with every overlay frame given as a JPEG ``path_to_image`` write the same files,
recorded images, third-party calls and JSON, with Pillow or the device encoders, and when the device declines a frame
(data after the scan's last MCU, which libjpeg skips with a warning)."""
import importlib.util
import json
import os
import tempfile

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _session_module():
    spec = importlib.util.spec_from_file_location('saver_session', os.path.join(ROOT, 'tests', 'golden',
                                                                                 'saver_session.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


ss = _session_module()
# the demo and gradio sessions with long ids, every overlay frame passed as a file
SESSIONS = [s for s in ss.SESSIONS if s[0] in ('demo', 'gradio') and s[1]]
SESSIONS = SESSIONS + [(d, li, v, p, [(ops, {('path' if k == 'image' else k): a for k, a in kw.items()})
                                      for ops, kw in frames]) for d, li, v, p, frames in SESSIONS]


def jpeg_writer(real_save, corrupt):
    """Writes the driver's path_to_image frames as JPEG (the file keeps its name); with corrupt, 3 bytes follow the
    scan's last MCU."""
    def save(img, p):
        real_save(img, p, format='JPEG', quality=90)
        if corrupt:
            data = open(p, 'rb').read()
            with open(p, 'wb') as f:
                f.write(data[:-2] + b'\x12\x34\x56' + data[-2:])
    return save


def replay(session, decoder, encoders, corrupt):
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference import result_utils

    def Saver(*a, **k):
        return result_utils.ResultSaver(*a, **k, png_encoder=encoders, jpeg_encoder=encoders, jpeg_decoder=decoder)
    rec = ss.Recorder()
    seeds = [(t + 3, t + 50) for t in range(len(session[4]))]
    real_save = Image.Image.save
    with rec.installed(), tempfile.TemporaryDirectory() as root:
        video_json = ss.drive(Saver, ObjectManager, ObjectInfo, session, seeds, root, rec,
                              jpeg_writer(real_save, corrupt), to_prob=lambda p: p.cuda())
        files = {}
        for d, _, names in os.walk(root):
            for n in names:
                files[os.path.relpath(os.path.join(d, n), root)] = open(os.path.join(d, n), 'rb').read()
    return json.loads(json.dumps(video_json)), rec.events, files


def same_events(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert len(x) == len(y)
        for u, v in zip(x, y):
            if isinstance(u, np.ndarray):
                assert u.dtype == v.dtype and np.array_equal(u, v)
            else:
                assert json.loads(json.dumps(u)) == json.loads(json.dumps(v))


@pytest.mark.parametrize('encoders', ['pil', 'device'])
@pytest.mark.parametrize('corrupt', [False, True])
@pytest.mark.parametrize('index', range(len(SESSIONS)))
def test_device_decoder_replays_pillow_path(index, encoders, corrupt):
    from deva.utils import jpeg_decode
    calls = []
    orig = jpeg_decode.decode_async

    def counted(hd):
        out = orig(hd)
        calls.append(out[1])
        return out
    want = replay(SESSIONS[index], 'pil', encoders, corrupt)
    jpeg_decode.decode_async = counted
    try:
        got = replay(SESSIONS[index], 'device', encoders, corrupt)
    finally:
        jpeg_decode.decode_async = orig
    assert got[0] == want[0]
    same_events(got[1], want[1])
    assert got[2].keys() == want[2].keys() and all(got[2][k] == want[2][k] for k in want[2])
    statuses = [int(s.item()) for s in calls]
    paths = sum(1 for _, kw in SESSIONS[index][4] if kw.get('path') and kw.get('save_the_mask', True))
    assert len(statuses) == paths  # every file-given overlay frame went to the device
    assert all((s != 0) == corrupt for s in statuses), statuses


def test_save_mask_with_device_decoder_does_not_synchronise():
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    om = ObjectManager()
    om.use_long_id = True
    om.add_new_objects([ObjectInfo(300, category_id=0, score=0.9), ObjectInfo(70000, category_id=1, score=0.5)])
    rec = ss.Recorder()
    with rec.installed() as real_save, tempfile.TemporaryDirectory() as root:
        p = os.path.join(root, 'frame.jpg')
        real_save(Image.fromarray(ss.make_image(5, ss.OUT)), p, format='JPEG')
        saver = ResultSaver(root, None, dataset='demo', object_manager=om, png_encoder='device',
                            jpeg_encoder='device', jpeg_decoder='device')
        prob = torch.from_numpy(ss.make_prob(5, 3)).cuda()
        for warm in (True, False):
            torch.cuda.synchronize()
            if not warm:
                torch.cuda.set_sync_debug_mode('error')
            try:
                for t in range(3):
                    saver.save_mask(prob, f'{t:05d}.jpg', need_resize=True, shape=ss.OUT, path_to_image=p)
                    saver.save_mask(prob, f'p{t:05d}.jpg', need_resize=True, shape=ss.OUT, path_to_image=p,
                                    prompts=ss.PROMPTS)
            finally:
                torch.cuda.set_sync_debug_mode('default')
        saver.end()
    assert [e[0] for e in rec.events].count('boxes') == 6
