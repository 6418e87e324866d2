"""``DeviceLoader`` against the same reader's host items, and its two new kernels (deva_b200_pil_resample_u8,
deva_b200_mask_nearest_ids) against the host oracle."""
import os
import sys

import numpy as np
import pytest
import torch
from torch.utils.data import default_collate

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
import reader_scenario as sc  # noqa: E402

pytestmark = pytest.mark.gpu

# the frames and masks the device reads in each run (the rest are declined files the host reads)
HOST_VOS = {3, 4, 5, 6}  # RGBA mask; progressive, greyscale and Exif JPEGs (with the 16-bit and interlaced masks)


@pytest.fixture(scope='module')
def clips(tmp_path_factory):
    from deva import _native
    _native.require_device()
    z = np.load(os.path.join(HERE, 'golden', 'readers.npz'))
    root = str(tmp_path_factory.mktemp('clips'))
    sc.materialise(sc.stored_files(z), root)
    return root


def _classes():
    from deva.inference.data.detection_video_reader import DetectionVideoReader
    from deva.inference.data.video_reader import VideoReader
    return {'VideoReader': VideoReader, 'DetectionVideoReader': DetectionVideoReader}


def _compare(got, want, resized, where):
    """got (the loader's item) equals want (the host item): structure, dtypes, devices, tolerances."""
    if isinstance(want, dict):
        assert isinstance(got, dict) and list(got) == list(want), (where, list(got), list(want))
        for k in want:
            _compare(got[k], want[k], resized, f'{where}/{k}')
    elif isinstance(want, (list, tuple)):
        assert type(got) is type(want) and len(got) == len(want), where
        for i, (g, w) in enumerate(zip(got, want)):
            _compare(g, w, resized, f'{where}/{i}')
    elif torch.is_tensor(want):
        device_side = where.endswith('/rgb') or where.endswith('/mask')
        assert got.is_cuda == device_side and got.dtype == want.dtype and got.shape == want.shape, \
            (where, got.device, got.dtype, got.shape, want.dtype, want.shape)
        if where.endswith('/rgb') and resized:
            err = float((got.cpu() - want).abs().max()) if want.numel() else 0.0
            assert err <= 1e-6, (where, err)
        else:
            assert torch.equal(got.cpu(), want), where
    else:
        assert type(got) is type(want) and got == want, (where, got, want)


def _host_items(reader):
    out = []
    for i in range(len(reader)):
        try:
            out.append(default_collate([reader[i]]))
        except Exception as e:  # noqa: BLE001
            out.append(e)
    return out


@pytest.mark.parametrize('run', sc.RUNS, ids=[r[0] for r in sc.RUNS])
@pytest.mark.parametrize('prefetch', [2, 16])
def test_loader_equals_reader(clips, run, prefetch):
    """Every run through ``DeviceLoader`` equals a second reader's sequential host pass, item for item, errors at the
    same index; declined files took the host path and eligible ones did not."""
    from deva.inference.data.device_loader import DeviceLoader
    try:
        host_reader = sc.make_reader(_classes(), run, clips)
    except Exception:  # noqa: BLE001  (a reader that cannot be built has nothing to load)
        return
    want = _host_items(host_reader)
    loader = DeviceLoader(sc.make_reader(_classes(), run, clips), prefetch=prefetch)
    assert len(loader) == len(want)
    it = iter(loader)
    for i, w in enumerate(want):
        if isinstance(w, Exception):
            with pytest.raises(type(w)) as e:
                next(it)
            assert str(e.value) == str(w), (run[0], i)
            return
        _compare(next(it), w, run[3]['size'] >= 0, f'{run[0]}/{i}')
    torch.cuda.synchronize()
    frames = list(loader.reader.frames)
    if run[2] == 'vos':  # frame 3's mask (RGBA) is read only with use_all_masks
        skip = set() if run[3].get('use_all_masks') else {3}
        host = {i for i, f in enumerate(frames) if int(f[:5]) in HOST_VOS - skip}
        assert set(loader.host_indices) == host, (run[0], loader.host_indices)
    elif run[2] in ('portrait', 'tiny', 'soft', 'det', 'bmx', 'vipseg'):
        assert loader.host_indices == [], run[0]


def test_one_jpeg_launch_per_window(clips, monkeypatch):
    """A window's JPEG frames go to one decode launch, its mask PNGs to one more."""
    from deva import _native
    from deva.inference.data.device_loader import DeviceLoader
    calls = {'jpeg': 0, 'png': 0}
    jpeg, png = _native.jpeg_decode, _native.png_decode

    def count(name, fn):
        def wrapped(*a):
            calls[name] += 1
            return fn(*a)
        return wrapped
    monkeypatch.setattr(_native, 'jpeg_decode', count('jpeg', jpeg))
    monkeypatch.setattr(_native, 'png_decode', count('png', png))
    run = next(r for r in sc.RUNS if r[0] == 'soft_multi_240')
    reader = sc.make_reader(_classes(), run, clips)
    items = list(DeviceLoader(reader, prefetch=4))
    assert len(items) == 3 and calls == {'jpeg': 2, 'png': 2}, calls


def test_bmx_frame_reproduces_ingest_fixture(clips):
    """The golden bmx-trees frame at size 240 gives ingest_vos240.npz's reference frame lattice and first mask."""
    from deva.inference.data.device_loader import DeviceLoader
    z = np.load(os.path.join(HERE, 'golden', 'ingest_vos240.npz'))
    item = next(iter(DeviceLoader(sc.make_reader(_classes(), next(r for r in sc.RUNS if r[0] == 'bmx_240'), clips))))
    rgb = item['rgb'][0].cpu()
    assert list(rgb.shape) == z['image0_shape'].tolist()
    assert float((rgb[:, ::8, ::8] - torch.from_numpy(z['image0_lattice'])).abs().max()) <= 1e-6
    assert torch.equal(item['mask'][0].cpu().to(torch.uint8), torch.from_numpy(z['mask0']))


@pytest.mark.parametrize('k', [1, 3, 40])
@pytest.mark.parametrize('shape', [(1, 1, 1, 1), (1, 1, 5, 7), (96, 160, 240, 400), (161, 97, 397, 240),
                                   (96, 160, 96, 300), (300, 7, 120, 7), (1080, 1920, 480, 853)])
def test_pil_resample_kernel_equals_oracle(k, shape):
    from deva.inference import frame_io
    from oracle import readers as oracle
    h, w, oh, ow = shape
    if k == 40 and h * w > 200000:
        k = 3
    planes = torch.from_numpy(np.random.default_rng(h * w + k).integers(0, 256, (k, h, w), dtype=np.uint8))
    out = torch.empty(k, oh, ow, device='cuda')
    # soft_from_u8 sizes its output like Resize(size); drive the tables directly for free (oh, ow)
    xb, xc = frame_io._axis_table('pil_bilinear', w, ow, 'cuda') if ow != w else (None, None)
    yb, yc = frame_io._axis_table('pil_bilinear', h, oh, 'cuda') if oh != h else (None, None)
    scratch = torch.empty(k, h, ow, dtype=torch.uint8, device='cuda')
    frame_io.nat.pil_resample_u8(planes.cuda(), k, h, w, oh, ow, xb, xc, yb, yc, scratch, out)
    got = out.cpu()
    for p in range(k):
        want = torch.from_numpy(oracle.pil_resample(planes[p].numpy(), oh, ow).astype(np.float32)) / 255
        assert torch.equal(got[p], want), (shape, p)


@pytest.mark.parametrize('channels', [1, 3])
@pytest.mark.parametrize('shape', [(1, 1, None), (17, 9, 480), (96, 160, 240), (1080, 1920, 480)])
def test_mask_ids_kernel_equals_oracle(channels, shape):
    from deva.inference import frame_io
    from oracle import readers as oracle
    h, w, size = shape
    rng = np.random.default_rng(h + channels)
    m = rng.integers(0, 256, (h, w, 3) if channels == 3 else (h, w), dtype=np.uint8)
    got = frame_io.mask_ids_from_u8(torch.from_numpy(m), size).cpu().numpy()
    oh, ow = (h, w) if size is None else frame_io.reader_size(h, w, size)
    rgb = m if channels == 3 else np.stack([m, np.zeros_like(m), np.zeros_like(m)], 2)
    np.testing.assert_array_equal(got, oracle.rgb_ids_nearest(rgb, oh, ow))
    assert got.dtype == np.int32


def test_loader_rejects_other_readers():
    from deva.inference.data.device_loader import DeviceLoader
    with pytest.raises(TypeError):
        DeviceLoader([1, 2, 3])
