"""Device side of the unsupervised DAVIS 2017 post-processing: deva_b200_label_areas against np.unique (1 and 3 / 4
channels, 1x1 to 1080p, 0 labels to more than the block-private table holds, exact and overflowing capacity, unaligned
frames), deva_b200_label_to_index against numpy, and the drop-in limit_max_id against every case of the unmodified
reference's outputs in tests/golden/unsup_davis17.{json,npz}: files, mode, palette, pixels, and the errors raised."""
import json
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import unsup_davis_scenario as us  # noqa: E402

pytestmark = pytest.mark.gpu
SHARED_SLOTS = 4096  # the block-private hash table of a colour frame (csrc/panoptic.cu)


def _labels(rng, h, w, n, channels):
    """Blocky labels from a pool of n non-zero labels plus 0, with 5 % per-pixel noise."""
    top = 255 if channels == 1 else (1 << 24) - 1
    pool = np.concatenate([[0], rng.choice(np.arange(1, top + 1), size=min(n, top), replace=False)]).astype(np.int64)
    bh, bw = max(1, h // 16), max(1, w // 16)
    blocks = rng.choice(pool, size=((h + bh - 1) // bh, (w + bw - 1) // bw))
    lab = np.repeat(np.repeat(blocks, bh, 0), bw, 1)[:h, :w]
    noise = rng.random((h, w)) < 0.05
    lab[noise] = rng.choice(pool, size=int(noise.sum()))
    return lab


def _frame(rng, lab, channels):
    if channels == 1:
        return lab.astype(np.uint8)
    planes = [lab >> 16, (lab >> 8) & 255, lab & 255] + ([rng.integers(0, 256, lab.shape)] if channels == 4 else [])
    return np.stack(planes, -1).astype(np.uint8)


def _on_device(a, offset):
    """a on the device at a byte offset from an aligned allocation (offset 1 takes the byte-load path)."""
    buf = torch.zeros(a.size + 4, dtype=torch.uint8, device='cuda')
    view = buf[offset:offset + a.size].view(a.shape)
    view.copy_(torch.from_numpy(a))
    return view


def _areas(frame, capacity):
    from deva import _native as nat
    labels = torch.full((capacity,), -5, dtype=torch.int32, device='cuda')  # the call initialises them
    counts, state = torch.full_like(labels, -5), torch.full((2,), -5, dtype=torch.int32, device='cuda')
    nat.label_areas(frame, labels, counts, state)
    return nat.label_areas_result(labels.cpu().numpy(), counts.cpu().numpy(), state.cpu().numpy())


@pytest.mark.parametrize('channels', [1, 3, 4])
@pytest.mark.parametrize('hw', [(1, 1), (7, 13), (480, 854), (1080, 1920)])
@pytest.mark.parametrize('n', [0, 1, 200, 6000])
def test_label_areas_matches_numpy(channels, hw, n):
    from deva import _native as nat
    nat.require_device()
    h, w = hw
    rng = np.random.default_rng(h * 31 + w + n + channels)
    lab = _labels(rng, h, w, n, channels)
    want_l, want_c = np.unique(lab[lab != 0], return_counts=True)
    if channels == 3 and n == 6000 and h == 1080:
        assert len(want_l) > SHARED_SLOTS  # the global-table path of labels that find no shared slot
    a = _frame(rng, lab, channels)
    for offset in (0, 1):
        for capacity in (max(len(want_l), 1), 2 * len(want_l) + 7):  # a full table and a roomy one
            got_l, got_c = _areas(_on_device(a, offset), capacity)
            order = np.argsort(got_l)
            np.testing.assert_array_equal(got_l[order], want_l)
            np.testing.assert_array_equal(got_c[order], want_c)


@pytest.mark.parametrize('channels', [1, 3])
def test_label_areas_capacity_overflow_raises(channels):
    from deva import _native as nat
    nat.require_device()
    rng = np.random.default_rng(5)
    lab = _labels(rng, 64, 96, 100, channels)
    distinct = len(np.unique(lab[lab != 0]))
    frame = _on_device(_frame(rng, lab, channels), 0)
    assert len(_areas(frame, distinct)[0]) == distinct
    with pytest.raises(RuntimeError, match='distinct labels'):
        _areas(frame, distinct - 1)


@pytest.mark.parametrize('channels', [1, 3, 4])
@pytest.mark.parametrize('hw', [(1, 1), (37, 53), (480, 854), (1080, 1920)])
def test_label_to_index_matches_numpy(channels, hw):
    from deva import _native as nat
    nat.require_device()
    h, w = hw
    rng = np.random.default_rng(h + w + channels)
    lab = _labels(rng, h, w, 120, channels)
    present = np.unique(lab)
    table = np.unique(np.concatenate([rng.choice(present, size=min(40, len(present)), replace=False),
                                      rng.integers(1, 256 if channels == 1 else 1 << 24, 20)])).astype(np.int32)
    index = rng.integers(0, 256, len(table)).astype(np.int32)
    i = np.minimum(np.searchsorted(table, lab), len(table) - 1)
    want = np.where(table[i] == lab, index[i], 0).astype(np.uint8)
    a = _frame(rng, lab, channels)
    for offset in (0, 1):
        out_buf = torch.full((h * w + 4,), 77, dtype=torch.uint8, device='cuda')
        out = out_buf[offset:offset + h * w].view(h, w)
        nat.label_to_index(_on_device(a, offset), torch.from_numpy(table).cuda(), torch.from_numpy(index).cuda(), out)
        np.testing.assert_array_equal(out.cpu().numpy(), want)
        assert (out_buf[:offset] == 77).all() and (out_buf[offset + h * w:] == 77).all()
    # an empty table maps every pixel to 0
    out = torch.full((h, w), 9, dtype=torch.uint8, device='cuda')
    empty = torch.zeros(0, dtype=torch.int32, device='cuda')
    nat.label_to_index(_on_device(a, 0), empty, empty, out)
    assert not out.any()


@pytest.fixture(scope='module')
def golden(golden_dir):
    return json.load(open(os.path.join(golden_dir, 'unsup_davis17.json'))), np.load(
        os.path.join(golden_dir, 'unsup_davis17.npz'))


@pytest.mark.parametrize('case', list(us.CASES))
def test_limit_max_id_matches_reference(golden, tmp_path, case):
    from deva.inference.postprocess_unsup_davis17 import limit_max_id
    meta, arrays = golden
    palette = bytes.fromhex(meta['palette'])
    error, files = us.run_case(lambda src, dst, m: limit_max_id(src, dst, m, palette=palette), str(tmp_path), case)
    us.assert_matches(meta, arrays, case, error, files)


def test_limit_max_id_many_labels_matches_oracle(tmp_path):
    """Frames with more distinct labels than the per-frame table (CAPACITY) are counted again with a larger one."""
    from deva.inference import postprocess_unsup_davis17 as pp
    from oracle import unsup_davis17 as ou
    rng = np.random.default_rng(3)
    os.makedirs(tmp_path / 'in' / 'v')
    for t in range(3):
        lab = rng.integers(0, 1 << 24, (48, 64 + t)) if t != 1 else rng.integers(0, 4, (48, 64))
        assert t == 1 or len(np.unique(lab)) > pp.CAPACITY
        Image.fromarray(_frame(rng, lab, 3)).save(tmp_path / 'in' / 'v' / f'{t}.png')
    palette = bytes(range(256)) * 3
    for m in (20, 255):
        pp.limit_max_id(str(tmp_path / 'in'), str(tmp_path / f'ours{m}'), m, palette=palette)
        ou.limit_max_id(str(tmp_path / 'in'), str(tmp_path / f'oracle{m}'), m, palette)
        ours, want = us.snapshot(str(tmp_path / f'ours{m}')), us.snapshot(str(tmp_path / f'oracle{m}'))
        assert sorted(ours) == sorted(want)
        for k in want:
            assert ours[k][:2] == want[k][:2]
            np.testing.assert_array_equal(ours[k][2], want[k][2])


def test_unsupported_mode_raises_value_error(tmp_path):
    from deva.inference.postprocess_unsup_davis17 import limit_max_id
    os.makedirs(tmp_path / 'in' / 'v')
    Image.fromarray(np.ones((8, 8), np.uint8)).save(tmp_path / 'in' / 'v' / '0.png')
    Image.new('LA', (8, 8)).save(tmp_path / 'in' / 'v' / '1.png')
    with pytest.raises(ValueError, match='1.png'):
        limit_max_id(str(tmp_path / 'in'), str(tmp_path / 'out'), 20, palette=bytes(768))
    assert not (tmp_path / 'out').exists()
