"""COCO compressed RLE (oracle/coco_rle.py, the format deva/utils/rle_encode.py writes on the device): hand-derived
cases from pycocotools' maskApi.c, round trips through the restated decoder on random, striped and single-pixel masks
and on 1x1, 1xW and Hx1 shapes, long runs and negative deltas, and pycocotools itself when it is installed.  Also the
package's encoder option, its input checks and its imports.  No GPU."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import coco_rle as oc

# (mask or counts, string), derived by hand from rleEncode / rleToString
MASKS = [
    (np.zeros((4, 4), np.uint8), [16], '`0'),  # 16 has bit 0x10 set: a second chunk
    (np.ones((4, 4), np.uint8), [0, 16], '0`0'),
    (np.array([[0, 1], [1, 1]], np.uint8), [1, 3], '13'),
    (np.array([[1, 0], [0, 0]], np.uint8), [0, 1, 3], '013'),
    (np.array([[1, 0], [1, 1], [0, 1]], np.uint8), [0, 2, 2, 2], '0220'),  # column-major
]
COUNTS = [
    ([1, 3, 2, 4], '1321'),  # i = 2 is not delta-coded
    ([5, 5, 5, 1], '555L'),  # delta -4
    ([1000, 20, 30, 5], 'Xo0d0n0A'),
    ([2073600], 'PPYo1'),  # an empty 1080p mask
]


@pytest.mark.parametrize('mask, cnts, string', MASKS)
def test_worked_masks(mask, cnts, string):
    assert oc.counts(mask) == cnts
    assert oc.encode(mask) == {'size': list(mask.shape), 'counts': string}
    assert list(oc.encode(mask)) == ['size', 'counts']
    np.testing.assert_array_equal(oc.decode(oc.encode(mask)), mask)


@pytest.mark.parametrize('cnts, string', COUNTS)
def test_worked_counts(cnts, string):
    assert oc.counts_to_string(cnts) == string
    assert oc.string_to_counts(string) == cnts


def _masks():
    rng = np.random.default_rng(0)
    out = []
    for h, w in [(1, 1), (1, 37), (41, 1), (7, 9), (64, 48), (120, 97)]:
        out.append(rng.random((h, w)) < 0.5)  # random
        out.append(rng.random((h, w)) < 0.03)  # sparse
        out.append(np.zeros((h, w), bool))
        out.append(np.ones((h, w), bool))
        stripes = np.zeros((h, w), bool)
        stripes[::2] = True  # alternates down every column
        out.append(stripes)
        cols = np.zeros((h, w), bool)
        cols[:, 1::3] = True  # whole-column runs
        out.append(cols)
        for y, x in [(0, 0), (h - 1, w - 1), (h // 2, w // 2), (0, w - 1), (h - 1, 0)]:
            single = np.zeros((h, w), bool)
            single[y, x] = True
            out.append(single)
    return out


@pytest.mark.parametrize('k', range(len(_masks())))
def test_round_trip(k):
    mask = _masks()[k]
    rle = oc.encode(mask)
    assert rle['size'] == list(mask.shape)
    assert sum(oc.string_to_counts(rle['counts'])) == mask.size
    np.testing.assert_array_equal(oc.decode(rle), mask.astype(np.uint8))


@pytest.mark.parametrize('run', [2**5, 2**5 - 1, 2**10, 2**10 + 3, 2**20, 2**20 + 7, 2**24 + 1])
def test_long_runs(run):
    """Runs whose chunk counts change at 2^4, 2^9, 2^19 and beyond, as counts and as deltas of either sign."""
    for cnts in ([run], [0, run], [run, 1, 1], [1, 1, 1, run], [run, run, 1, 1, run, 1], [1, run, run, 1, 1, 1]):
        s = oc.counts_to_string(cnts)
        assert oc.string_to_counts(s) == cnts, (cnts, s)
    mask = np.zeros((run + 3, 1), bool)
    mask[2:2 + run] = True
    assert oc.counts(mask) == [2, run, 1]
    np.testing.assert_array_equal(oc.decode(oc.encode(mask)), mask)


def test_negative_deltas():
    cnts = [3, 900, 40, 2, 1, 70000, 5, 1, 1, 1]
    s = oc.counts_to_string(cnts)
    assert oc.string_to_counts(s) == cnts
    # the sign-terminated chunks: -4 is one chunk ('L' = 48 + 28), -17 needs two
    assert oc.counts_to_string([5, 5, 5, 1]).endswith('L')
    assert len(oc.counts_to_string([1, 20, 1, 3])) == 1 + 2 + 1 + 2  # 3 - 20 = -17


def test_string_length_bound():
    """Every mask's string is at most h * w + 1 characters (deva_b200_rle_bound per entry): the longest is the one
    whose value changes at every pixel."""
    rng = np.random.default_rng(1)
    for h, w in [(1, 1), (1, 2), (3, 5), (16, 17), (33, 64)]:
        alt = (np.arange(h * w).reshape((h, w), order='F') % 2).astype(bool)
        for mask in (alt, ~alt, rng.random((h, w)) < 0.5, np.zeros((h, w), bool)):
            assert len(oc.encode(mask)['counts']) <= h * w + 1
        assert len(oc.encode(~alt)['counts']) == h * w + 1


def test_encode_ids_matches_per_mask_encode():
    ids = np.random.default_rng(2).integers(-2, 5, (13, 17)) * (2**62 // 4)
    seg = [0, 2**62 // 4, 2**62 // 4, 7, -2 * (2**62 // 4)]
    assert oc.encode_ids(ids, seg) == [oc.encode(ids == i) for i in seg]
    assert oc.encode_ids(ids, [7])[0]['counts'] == oc.counts_to_string([13 * 17])


def test_matches_pycocotools():
    mask_util = pytest.importorskip('pycocotools.mask')
    rng = np.random.default_rng(3)
    for h, w in [(1, 1), (1, 50), (50, 1), (37, 61), (270, 481)]:
        for p in (0.0, 0.02, 0.5, 1.0):
            m = rng.random((h, w)) < p
            want = mask_util.encode(np.asfortranarray(m))
            want['counts'] = want['counts'].decode('utf-8')
            assert oc.encode(m) == want


# ---------------------------------------------------------------------------------------------- package surface
def test_resolve_encoder(monkeypatch):
    from deva.utils.rle_encode import resolve_encoder
    monkeypatch.delenv('DEVA_B200_RLE_ENCODER', raising=False)
    assert resolve_encoder() == 'pycocotools'
    assert resolve_encoder('device') == 'device'
    monkeypatch.setenv('DEVA_B200_RLE_ENCODER', 'device')
    assert resolve_encoder() == 'device'
    assert resolve_encoder('pycocotools') == 'pycocotools'
    with pytest.raises(ValueError, match='rle_encoder'):
        resolve_encoder('cpu')


def test_saver_reads_the_encoder_option(monkeypatch):
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    monkeypatch.delenv('DEVA_B200_RLE_ENCODER', raising=False)
    for arg, env, want in [(None, None, 'pycocotools'), ('device', None, 'device'), (None, 'device', 'device'),
                           ('pycocotools', 'device', 'pycocotools')]:
        if env is not None:
            monkeypatch.setenv('DEVA_B200_RLE_ENCODER', env)
        saver = ResultSaver('/nonexistent', 'ds/seq', dataset='burst', object_manager=ObjectManager(), rle_encoder=arg)
        assert saver.rle_encoder == want
        saver.end()
    with pytest.raises(ValueError, match='rle_encoder'):
        ResultSaver('/nonexistent', 'ds/seq', dataset='burst', object_manager=ObjectManager(), rle_encoder='cpu')


def test_bad_inputs_raise():
    """Checked on the host, before anything reaches the device."""
    from deva.utils.rle_encode import MAX_SEGMENT_CHANNELS, encode_rle_async
    ids = np.zeros((4, 5), np.int64)
    for bad in (np.zeros((4, 5, 2), np.int64), np.zeros(7, np.int64), ids.astype(np.float32), ids.astype(np.uint64),
                np.zeros((0, 5), np.int64), np.zeros((5, 0), np.int64), [[1, 2], [3, 4]]):
        with pytest.raises(ValueError):
            encode_rle_async(bad, [1])
    for seg in ([1.5], [2**63], [-2**63 - 1], ['a'], [True], list(range(MAX_SEGMENT_CHANNELS + 1))):
        with pytest.raises(ValueError):
            encode_rle_async(ids, seg)


def test_too_many_pixels_raise():
    from deva.utils.rle_encode import encode_rle_async
    big = np.broadcast_to(np.int8(0), (2**16, 2**15))  # 2^31 pixels, never materialised: the shape alone fails
    with pytest.raises(ValueError, match='2\\^31'):
        encode_rle_async(big, [1])


def test_import_without_pycocotools_does_not_initialise_cuda():
    code = ('import sys; sys.modules["pycocotools"] = None; sys.modules["pycocotools.mask"] = None\n'
            'import torch, deva.utils.rle_encode, deva.inference.result_utils\n'
            'assert not torch.cuda.is_initialized()\n'
            'assert sys.modules["pycocotools"] is None')
    subprocess.run([sys.executable, '-c', code], check=True, cwd=os.path.dirname(os.path.abspath(__file__)),
                   env={**os.environ, 'PYTHONPATH': os.pathsep.join(sys.path)})
