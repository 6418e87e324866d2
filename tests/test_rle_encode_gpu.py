"""COCO RLE encoded on the device (csrc/rle.cu, deva/utils/rle_encode.py): string for string oracle/coco_rle.py's over
1x1, 1xW, Hx1, 270x481, 720p and 1080p maps (constant maps, ellipses with up to 300 ids, salt-and-pepper noise, the
map that changes id at every pixel, checkerboards, first and last pixel set, ids near +-2^62) with duplicate, absent
and up to MAX_SEGMENT_CHANNELS seg ids; deterministic, within deva_b200_rle_bound, and enqueued without a host
synchronisation.  In the result saver with rle_encoder='device': the recorded burst session of tests/golden/saver.json
with each recorded mask's oracle string, and further burst sessions equal to the default pycocotools path with
pycocotools.mask.encode bound to the oracle."""
import contextlib
import functools
import json
import os
import sys
import tempfile
import types

import numpy as np
import pytest
import torch

from oracle import coco_rle as oc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
BIG = 2**62


def ellipses(h, w, k, seed=0, ids=None):
    """int64 [h, w]: 0 under k random ellipses, later ones covering earlier ones; ellipse i carries ids[i] (i + 1)."""
    rng = np.random.default_rng(seed)
    out = np.zeros((h, w), np.int64)
    yy, xx = np.mgrid[:h, :w]
    for i in range(k):
        cy, cx = rng.uniform(0, h), rng.uniform(0, w)
        ay, ax = rng.uniform(1, max(2, h / 4)), rng.uniform(1, max(2, w / 4))
        out[((yy - cy) / ay)**2 + ((xx - cx) / ax)**2 <= 1] = i + 1 if ids is None else ids[i]
    return out


def every_pixel(h, w, values=(3, 8)):
    """The map whose id changes at every pixel of the column-major scan (the bound's worst case)."""
    order = np.arange(h * w).reshape((h, w), order='F')
    return np.asarray(values, np.int64)[order % len(values)]


def make_map(kind, h, w):
    rng = np.random.default_rng(h * 7919 + w)
    if kind == 'constant':
        return np.full((h, w), 4, np.int64)
    if kind == 'zero':
        return np.zeros((h, w), np.int64)
    if kind.startswith('ellipses'):
        return ellipses(h, w, int(kind[8:]), seed=h + w)
    if kind == 'noise':
        return rng.choice(np.array([0, 1, 2], np.int64), (h, w))
    if kind == 'every_pixel':
        return every_pixel(h, w)
    if kind == 'checker':
        return ((np.arange(h)[:, None] + np.arange(w)[None]) % 2).astype(np.int64) * 6
    if kind == 'first_last':
        m = np.zeros((h, w), np.int64)
        m[0, 0] = m[-1, -1] = 5
        return m
    if kind == 'big_ids':
        return ellipses(h, w, 6, seed=5, ids=[BIG, BIG - 1, -BIG, -BIG + 1, 2**63 - 1, -2**63])
    raise ValueError(kind)


def seg_list(ids, extra_absent=True):
    present = [int(v) for v in np.unique(ids)]
    seg = present + present[:2]  # duplicates
    if extra_absent:
        seg += [123456789, -1 if -1 not in present else -7]
    return np.random.default_rng(len(seg)).permutation(np.array(seg, dtype=object)).tolist()


def want(ids, seg):
    cache = {}
    present = set(np.unique(ids).tolist())
    empty = oc.counts_to_string([ids.size])
    for i in seg:
        if i not in cache:
            cache[i] = oc.encode(ids == i)['counts'] if i in present else empty
    return [{'size': list(ids.shape), 'counts': cache[i]} for i in seg]


SMALL = [(1, 1), (1, 97), (89, 1), (270, 481)]
KINDS = ['constant', 'zero', 'ellipses5', 'ellipses60', 'noise', 'every_pixel', 'checker', 'first_last', 'big_ids']
CASES = [(k, h, w) for h, w in SMALL for k in KINDS]
CASES += [(k, 720, 1280) for k in ('constant', 'ellipses10', 'ellipses300', 'checker', 'first_last', 'big_ids')]
CASES += [(k, 1080, 1920) for k in ('ellipses50', 'ellipses300', 'noise', 'every_pixel', 'first_last')]


@pytest.mark.parametrize('kind, h, w', CASES)
def test_device_matches_oracle(kind, h, w):
    from deva import _native
    from deva.utils.rle_encode import encode_rle_async
    ids = make_map(kind, h, w)
    seg = seg_list(ids)
    dev = torch.from_numpy(ids).cuda()
    pending = encode_rle_async(dev, seg)
    got = pending.result()
    assert got == want(ids, seg), (kind, h, w)
    total = sum(len(r['counts']) for r in got)
    assert total <= _native.rle_bound(h, w, len(seg))
    assert encode_rle_async(dev, seg).result() == got  # repeated encodes are identical


def test_every_pixel_reaches_the_bound():
    """A mask that changes at every pixel and starts set: h * w + 1 characters, the per-entry bound."""
    from deva import _native
    from deva.utils.rle_encode import encode_rle
    h, w = 37, 53
    ids = every_pixel(h, w, (9, 2))
    got = encode_rle(torch.from_numpy(ids).cuda(), [9, 9, 2])
    assert [len(r['counts']) for r in got] == [h * w + 1, h * w + 1, h * w]
    assert sum(len(r['counts']) for r in got) <= _native.rle_bound(h, w, 3)
    assert got == want(ids, [9, 9, 2])


@pytest.mark.parametrize('shape', [(270, 481), (64, 64)])
def test_max_segment_channels(shape):
    """n = MAX_SEGMENT_CHANNELS: every present id, duplicates and absent ids, in a shuffled order."""
    from deva import _native
    from deva.utils.rle_encode import encode_rle
    h, w = shape
    ids = ellipses(h, w, 300, seed=3)
    present = [int(v) for v in np.unique(ids)]
    rng = np.random.default_rng(0)
    seg = present + rng.integers(-10**6, 10**6, _native.MAX_SEGMENT_CHANNELS - len(present)).tolist()
    seg = rng.permutation(np.array(seg, dtype=object)).tolist()
    seg[-1] = seg[0]
    assert len(seg) == _native.MAX_SEGMENT_CHANNELS
    assert encode_rle(torch.from_numpy(ids).cuda(), seg) == want(ids, seg)


def test_long_runs_and_many_chunks():
    """A tall single column (runs of 2^20 and more, boundaries in the first and last chunk) and a wide row."""
    from deva.utils.rle_encode import encode_rle
    col = np.zeros((3 * 2**20 + 5, 1), np.int64)
    col[7:7 + 2**20] = 1
    col[-3:] = 2
    assert encode_rle(torch.from_numpy(col).cuda(), [0, 1, 2, 3]) == want(col, [0, 1, 2, 3])
    row = np.zeros((1, 2**20 + 33), np.int64)
    row[0, ::4097] = 5
    assert encode_rle(torch.from_numpy(row).cuda(), [5, 0]) == want(row, [5, 0])


def test_inputs_of_other_forms():
    """numpy maps, narrower integer dtypes, strided CUDA views and seg ids as arrays or tensors give the same strings;
    an empty seg list gives an empty list."""
    from deva.utils.rle_encode import encode_rle
    ids = ellipses(61, 85, 12, seed=9)
    seg = [int(v) for v in np.unique(ids)] + [99]
    base = want(ids, seg)
    assert encode_rle(ids, seg) == base
    assert encode_rle(ids.astype(np.int16), np.array(seg)) == base
    assert encode_rle(torch.from_numpy(ids).cuda().to(torch.int32), torch.tensor(seg)) == base
    wide = torch.from_numpy(np.repeat(ids, 2, axis=1)).cuda()
    assert encode_rle(wide[:, ::2], seg) == base
    assert encode_rle(torch.from_numpy(ids).cuda(), []) == []


def test_rejects_bad_inputs():
    from deva.utils.rle_encode import encode_rle
    for bad in (torch.zeros(4, 5, dtype=torch.float32, device='cuda'), torch.zeros(4, 5, dtype=torch.int64),
                torch.zeros(2, 4, 5, dtype=torch.int64, device='cuda'), torch.zeros(0, 5, dtype=torch.int64,
                                                                                   device='cuda')):
        with pytest.raises(ValueError):
            encode_rle(bad, [1])
    with pytest.raises(ValueError):
        encode_rle(torch.zeros(4, 5, dtype=torch.int64, device='cuda'), torch.tensor([1], device='cuda'))


def test_encode_async_does_not_synchronise():
    from deva.utils.rle_encode import encode_rle_async, host_bytes
    ids = torch.from_numpy(ellipses(1080, 1920, 50, seed=1)).cuda()
    seg = list(range(51))
    encode_rle_async(ids, seg).result()  # warm the allocator and the library
    host = torch.empty(host_bytes(len(seg)), dtype=torch.uint8, pin_memory=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        pending = encode_rle_async(ids, seg, host=host)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert pending.result() == want(ids.cpu().numpy(), seg)


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


def test_saver_replay_burst_with_device_rle(saver_fixture):
    """The recorded burst session with rle_encoder='device': the JSON as recorded with each stub counts
    ("{sum}:{digest}") replaced by the oracle's string of the recorded mask, every PNG event as recorded, no RLE
    event (pycocotools is not called)."""
    ss, meta, arrays = saver_fixture
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    index = [k for k, s in enumerate(ss.SESSIONS) if s[0] == 'burst']
    assert index == [1]
    expected = meta['sessions'][1]
    strings = {}
    for e in expected['events']:
        if e[0] == 'rle':
            m = arrays[e[-1]]
            strings[f'{int(m.sum())}:{ss.digest(np.packbits(m))}'] = oc.encode(m)['counts']
    assert strings
    want_json = json.loads(json.dumps(expected['video_json']))
    n = 0
    for frame in want_json['segmentations']:
        for s in frame['segmentations']:
            s['rle']['counts'] = strings[s['rle']['counts']]
            n += 1
    assert n > 0
    rec = ss.Recorder()
    with rec.installed() as orig_save, tempfile.TemporaryDirectory() as root:
        video_json = ss.drive(functools.partial(ResultSaver, rle_encoder='device'), ObjectManager, ObjectInfo,
                              ss.SESSIONS[1], expected['seeds'], root, rec, orig_save, to_prob=lambda p: p.cuda())
    assert json.loads(json.dumps(video_json)) == want_json
    rest = [e for e in expected['events'] if e[0] != 'rle']
    assert [e[0] for e in rec.events] == [e[0] for e in rest] and all(e[0] == 'image' for e in rest)
    for got, w in zip(rec.events, rest):
        assert list(got[:-1]) == w[:-1]
        assert np.array_equal(got[-1], arrays[w[-1]]), w


@contextlib.contextmanager
def pycocotools_for(encoder):
    """For 'pycocotools': pycocotools.mask.encode bound to the oracle (bytes counts, as pycocotools returns them); for
    'device': pycocotools made unimportable."""
    coco = types.ModuleType('pycocotools')
    coco.mask = types.ModuleType('pycocotools.mask')

    def encode(m):
        assert m.flags['F_CONTIGUOUS'] and m.ndim == 2
        return {'size': list(m.shape), 'counts': oc.encode(m)['counts'].encode()}

    coco.mask.encode = encode
    saved = {k: sys.modules.get(k) for k in ('pycocotools', 'pycocotools.mask')}
    if encoder == 'pycocotools':
        sys.modules.update({'pycocotools': coco, 'pycocotools.mask': coco.mask})
    else:
        sys.modules.update({'pycocotools': None, 'pycocotools.mask': None})
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def _many(t):
    ops = [('add', [(100 + 3 * t + j, j % 3, 0.3 + 0.01 * j) for j in range(3)])]
    if t % 3 == 2:
        ops.append(('del', [100 + 3 * (t - 2), 100 + 3 * (t - 1) + 1]))
    return ops


# dataset, use_long_id, video_name, palette, frames: as tests/golden/saver_session.py's SESSIONS
EXTRA_SESSIONS = [
    ('burst', True, 'ds/long_ids', None, [
        ([('add', [(1234567, 0, 0.9), (70000, 1, 0.8), (300, 2, 0.75), (2**24 - 1, 0, 0.5)])], dict(resize=True)),
        ([('del', [70000]), ('add', [(4096, 1, 0.6)])], dict(resize=False)),
        ([], dict(resize=True)),
    ]),
    # 50+ objects: later rectangles cover earlier ones, so many segments have zero area and are dropped
    ('burst', False, 'ds/many', None, [
        ([('add', [(i, i % 3, 0.5 + 0.001 * i) for i in range(1, 56)])], dict(resize=True)),
        ([('del', list(range(1, 20, 2)))], dict(resize=False)),
        ([('add', [(200 + i, 0, 0.4) for i in range(12)])], dict(resize=True)),
    ]),
    # longer than the ring of pinned slots (12), objects changing while frames are queued, resize and no resize
    ('burst', False, 'ds/queued', None, [(_many(t), dict(resize=t % 2 == 0)) for t in range(18)]),
    ('burst', False, 'ds/empty', None, [([], dict(resize=True)), ([('add', [(5, 0, 0.5)])], dict())]),
]


@pytest.mark.parametrize('index', range(len(EXTRA_SESSIONS)))
def test_saver_sessions_match_default_path(saver_fixture, index):
    """Each session's JSON with rle_encoder='device' (pycocotools unimportable) equals the default path's with the
    oracle as pycocotools; the PNGs are the same files."""
    ss = saver_fixture[0]
    from PIL import Image
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    session = EXTRA_SESSIONS[index]
    seeds = [(1000 * index + t, t) for t in range(len(session[4]))]
    out = {}
    for enc in ('pycocotools', 'device'):
        with pycocotools_for(enc), tempfile.TemporaryDirectory() as root:
            video_json = ss.drive(functools.partial(ResultSaver, rle_encoder=enc), ObjectManager, ObjectInfo, session,
                                  seeds, root, ss.Recorder(), Image.Image.save, to_prob=lambda p: p.cuda())
            pngs = {os.path.relpath(os.path.join(d, f), root): open(os.path.join(d, f), 'rb').read()
                    for d, _, fs in os.walk(root) for f in fs}
        out[enc] = (json.loads(json.dumps(video_json)), pngs)
    assert out['device'][0] == out['pycocotools'][0]
    assert out['device'][1] == out['pycocotools'][1]
    frames = out['device'][0]['segmentations']
    assert len(frames) == len(session[4])
    if index == 1:  # zero-area segments were dropped
        assert len(frames[0]['segmentations']) < 55


def test_save_mask_with_device_rle_does_not_synchronise(saver_fixture):
    """Burst-mode save_mask with rle_encoder='device' enqueues its work without a host synchronisation and leaves the
    id map on the device; the JSON equals the default path's with the oracle as pycocotools."""
    ss = saver_fixture[0]
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    om = ObjectManager()
    om.add_new_objects([ObjectInfo(i, category_id=i % 3, score=0.5) for i in range(1, 8)])
    prob = torch.from_numpy(ss.make_prob(5, 8)).cuda()
    outputs = {}
    for enc in ('pycocotools', 'device'):
        with pycocotools_for(enc), tempfile.TemporaryDirectory() as root:
            saver = ResultSaver(root, 'ds/seq', dataset='burst', object_manager=om, rle_encoder=enc)
            saver.save_mask(prob, '00000.jpg', need_resize=True, shape=ss.OUT)  # warm up
            saver.queue.join()
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode('error' if enc == 'device' else 'default')
            try:
                for t in range(1, 4):
                    saver.save_mask(prob, f'{t:05d}.jpg', need_resize=True, shape=ss.OUT)
            finally:
                torch.cuda.set_sync_debug_mode('default')
            saver.end()
            slots = list(saver.free_slots.queue)
            outputs[enc] = json.loads(json.dumps(saver.video_json))
        if enc == 'device':
            assert all('ids' not in slot for slot in slots)
            assert any('rle' in slot for slot in slots)
    assert outputs['device'] == outputs['pycocotools']
    assert len(outputs['device']['segmentations']) == 4
