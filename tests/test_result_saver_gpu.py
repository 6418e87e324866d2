"""Result saver on the device (deva/inference/result_utils.py, frame_io.prob_to_segments) against the reference's
ResultSaver (tests/golden/saver.{json,npz}, minted by make_saver_golden.py) and against torch."""
import importlib.util
import json
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _session_module(golden_dir):
    spec = importlib.util.spec_from_file_location('saver_session', os.path.join(golden_dir, 'saver_session.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module')
def fixture(golden_dir):
    meta = json.load(open(os.path.join(golden_dir, 'saver.json')))
    return _session_module(golden_dir), meta, np.load(os.path.join(golden_dir, 'saver.npz'))


@pytest.mark.parametrize('index', range(8))
def test_replay_matches_reference(fixture, index):
    """Every recorded image (path, mode, palette, pixels), RLE input, supervision call, gradio frame and the JSON."""
    ss, meta, arrays = fixture
    assert len(ss.SESSIONS) == len(meta['sessions']) == 8
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    expected = meta['sessions'][index]
    rec = ss.Recorder()
    with rec.installed() as orig_save, tempfile.TemporaryDirectory() as root:
        video_json = ss.drive(ResultSaver, ObjectManager, ObjectInfo, ss.SESSIONS[index], expected['seeds'], root, rec,
                              orig_save, to_prob=lambda p: p.cuda())
    assert json.loads(json.dumps(video_json)) == expected['video_json']
    assert len(rec.events) == len(expected['events'])
    for got, want in zip(rec.events, expected['events']):
        if isinstance(got[-1], np.ndarray):
            ref = arrays[want[-1]]
            assert list(got[:-1]) == want[:-1], (got[:-1], want[:-1])
            assert got[-1].dtype == ref.dtype and got[-1].shape == ref.shape, (want, got[-1].dtype, got[-1].shape)
            assert np.array_equal(got[-1], ref), (want, int((got[-1] != ref).sum()))
        else:
            assert json.loads(json.dumps(list(got))) == want


def _random_prob(c, h, w, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    prob = torch.softmax(3 * torch.randn(c, (h + 7) // 8, (w + 7) // 8, device='cuda', generator=g), 0)
    return F.interpolate(prob.unsqueeze(0), size=(h, w), mode='bilinear', align_corners=False)[0].contiguous()


@pytest.mark.parametrize('c', [1, 2, 201, 4096])
@pytest.mark.parametrize('size', [None, (97, 131)])
def test_prob_to_segments_matches_torch(c, size):
    from deva.inference.frame_io import id_rgb, prob_to_ids, prob_to_segments
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from torchvision.ops import masks_to_boxes
    h, w = 61, 85
    prob = _random_prob(c, h, w, seed=c)
    om = ObjectManager()
    om.use_long_id = True
    om.add_new_objects([ObjectInfo(256 + 977 * i) for i in range(1, c)])
    if c > 3:
        om.delete_object([256 + 977 * 2])  # the last channel keeps no object: id 0, not coloured
    oh, ow = (h, w) if size is None else size
    g = torch.Generator(device='cuda').manual_seed(7)
    frame = torch.randint(0, 256, (oh, ow, 3), device='cuda', dtype=torch.uint8, generator=g)
    seg = prob_to_segments(prob, om, size, index=True, rgb=True, frame=frame, stats=True)
    lut = torch.tensor(seg.lut, dtype=torch.int32, device='cuda')
    ids = prob_to_ids(prob, size=size, lut=lut)
    channel = prob_to_ids(prob, size=size)
    assert torch.equal(seg.index, ids.to(torch.uint8))
    assert torch.equal(seg.counts, torch.bincount(channel.flatten(), minlength=c))
    present = torch.nonzero(seg.counts).flatten()
    masks = channel[None] == present[:, None, None]
    assert torch.equal(seg.boxes[present].float(), masks_to_boxes(masks))
    absent = seg.counts == 0
    assert torch.equal(seg.boxes[absent], torch.tensor([2**31 - 1, 2**31 - 1, -1, -1], dtype=torch.int32,
                                                       device='cuda').expand(int(absent.sum()), 4))
    # numpy formulas of the reference's saver (result_utils.py:208-215, 240-242)
    ids_np, frame_np = ids.cpu().numpy(), frame.cpu().numpy()
    rgb_np = np.zeros((oh, ow, 3), np.uint8)
    for obj in om.obj_to_tmp_id:
        rgb_np[ids_np == obj.id] = [(obj.id >> s) & 255 for s in (0, 8, 16)]
        assert id_rgb(obj.id) == int.from_bytes(bytes([(obj.id >> s) & 255 for s in (0, 8, 16)]), 'little')
    alpha = (ids_np == 0).astype(np.float32)[:, :, None] * 0.5 + 0.5
    blend = (frame_np * alpha + rgb_np * (1 - alpha)).astype(np.uint8)
    assert np.array_equal(seg.rgb.cpu().numpy(), rgb_np)
    assert np.array_equal(seg.overlay.cpu().numpy(), blend)


def test_prob_to_segments_rejects_too_many_channels():
    from deva import _native as nat
    from deva.inference.frame_io import prob_to_segments
    from deva.inference.object_manager import ObjectManager
    prob = torch.rand(nat.MAX_SEGMENT_CHANNELS + 1, 4, 5, device='cuda')
    with pytest.raises(RuntimeError, match='channels'):
        prob_to_segments(prob, ObjectManager(), stats=True)


def test_save_mask_does_not_synchronise(fixture):
    """The device path (uint8 frame, overlay, prompts, JSON) enqueues its work without a host synchronisation."""
    ss = fixture[0]
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    om = ObjectManager()
    om.use_long_id = True
    om.add_new_objects([ObjectInfo(300, category_id=0, score=0.9), ObjectInfo(70000, category_id=1, score=0.5)])
    rec = ss.Recorder()
    with rec.installed(), tempfile.TemporaryDirectory() as root:
        saver = ResultSaver(root, None, dataset='demo', object_manager=om)
        prob = torch.from_numpy(ss.make_prob(5, 3)).cuda()
        image = ss.make_image(5, ss.OUT)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            for t in range(3):
                saver.save_mask(prob, f'{t:05d}.jpg', need_resize=True, shape=ss.OUT, image_np=image,
                                prompts=ss.PROMPTS)
        finally:
            torch.cuda.set_sync_debug_mode('default')
        saver.end()
    assert [e[0] for e in rec.events].count('image') == 6
