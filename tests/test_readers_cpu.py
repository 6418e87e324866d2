"""The drop-in dataset readers (deva/inference/data/) against the reference readers' fixture, and the host oracle of
their mask transforms against Pillow.  No GPU needed."""
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch
from PIL import Image
from torch.utils.data import DataLoader, default_collate

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PKG = os.path.join(ROOT, 'tracking-anything-with-deva_b200')
sys.path.insert(0, os.path.join(HERE, 'golden'))
import reader_scenario as sc  # noqa: E402

from deva.inference.data.detection_video_reader import DetectionVideoReader  # noqa: E402
from deva.inference.data.video_reader import VideoReader  # noqa: E402
from oracle import readers as oracle  # noqa: E402

CLASSES = {'VideoReader': VideoReader, 'DetectionVideoReader': DetectionVideoReader}


@pytest.fixture(scope='module')
def golden(tmp_path_factory):
    z = np.load(os.path.join(HERE, 'golden', 'readers.npz'))
    meta = json.load(open(os.path.join(HERE, 'golden', 'readers.json')))
    root = str(tmp_path_factory.mktemp('clips'))
    sc.materialise(sc.stored_files(z), root)
    return z, meta, root


def assert_matches(value, rec, z, root, where):
    """``value`` (a collated item or part of one) equals the fixture record ``rec``: structure, types, dtypes, shapes
    and values, bit for bit."""
    if 'dict' in rec:
        assert isinstance(value, dict) and list(value) == [k for k, _ in rec['dict']], (where, list(value))
        for k, r in rec['dict']:
            assert_matches(value[k], r, z, root, f'{where}/{k}')
    elif 'list' in rec or 'tuple' in rec:
        items = rec.get('list', rec.get('tuple'))
        assert type(value).__name__ == ('list' if 'list' in rec else 'tuple') and len(value) == len(items), where
        for i, r in enumerate(items):
            assert_matches(value[i], r, z, root, f'{where}/{i}')
    elif 'str' in rec:
        assert isinstance(value, str) and value.replace(root, sc.ROOT_TOKEN) == rec['str'], (where, value)
    elif 'tensor' in rec:
        assert torch.is_tensor(value) and str(value.dtype) == rec['tensor'] and list(value.shape) == rec['shape'], \
            (where, value.dtype, value.shape, rec)
        t = value.detach().cpu()
        if 'sha256' in rec:
            assert sc.digest(t) == rec['sha256'], (where, 'sum', float(t.double().sum()), 'expected', rec['sum'])
        else:
            np.testing.assert_array_equal(t.numpy(), z[rec['key']], err_msg=where)
    else:
        (kind, v), = rec.items()
        assert type(value).__name__ == kind and value == v, (where, value, rec)


@pytest.mark.parametrize('run', sc.RUNS, ids=[r[0] for r in sc.RUNS])
def test_reader_equals_reference(golden, run):
    """Item for item, ``default_collate([reader[i]])`` equals the reference reader's, errors included."""
    z, meta, root = golden
    want = meta['runs'][run[0]]
    if 'init_error' in want:
        with pytest.raises(Exception) as e:
            sc.make_reader(CLASSES, run, root)
        assert sc.error_record(e.value, root) == want['init_error']
        return
    reader = sc.make_reader(CLASSES, run, root)
    assert len(reader) == want['len']
    for i, rec in enumerate(want['items']):
        try:
            item = default_collate([reader[i]])
        except Exception as e:  # noqa: BLE001
            assert sc.error_record(e, root) == rec, (run[0], i)
            continue
        assert 'error' not in rec, (run[0], i, rec)
        assert_matches(item, rec, z, root, f'{run[0]}/{i}')


@pytest.mark.parametrize('name', ['vos_all_240', 'soft_multi_240'])
def test_reader_in_dataloader_workers(golden, name):
    """The drivers' ``DataLoader(reader, batch_size=1, num_workers=2)`` yields the fixture's items.  (Not for
    ``DetectionVideoReader``: its ``is_rgb`` carries over within each worker, so there, as in the reference, items
    depend on how the workers share them.)"""
    z, meta, root = golden
    run = next(r for r in sc.RUNS if r[0] == name)
    reader = sc.make_reader(CLASSES, run, root)
    items = list(DataLoader(reader, batch_size=1, shuffle=False, num_workers=2))
    assert len(items) == meta['runs'][name]['len']
    for i, (item, rec) in enumerate(zip(items, meta['runs'][name]['items'])):
        assert_matches(item, rec, z, root, f'{name}/{i}')


def test_oracle_resample_equals_pillow():
    """oracle.pil_resample == Image.resize(BILINEAR) of an L image: down, up, mixed, one axis, 4000 -> 1."""
    hyp = pytest.importorskip('hypothesis')
    st = hyp.strategies

    @hyp.settings(max_examples=150, deadline=None, derandomize=True)
    @hyp.given(st.integers(1, 300), st.integers(1, 300), st.integers(1, 300), st.integers(1, 300), st.integers(0, 99))
    def check(h, w, oh, ow, seed):
        img = np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)
        want = np.asarray(Image.fromarray(img).resize((ow, oh), Image.BILINEAR))
        np.testing.assert_array_equal(oracle.pil_resample(img, oh, ow), want)
    check()
    for h, w, oh, ow in ((4000, 3, 1, 3), (3, 4000, 3, 1), (1, 1, 7, 5), (97, 161, 97, 300), (161, 97, 40, 97)):
        img = np.random.default_rng(h).integers(0, 256, (h, w), dtype=np.uint8)
        want = np.asarray(Image.fromarray(img).resize((ow, oh), Image.BILINEAR))
        np.testing.assert_array_equal(oracle.pil_resample(img, oh, ow), want)


def test_package_coefficients_equal_oracle():
    """frame_io.pil_bilinear_coeffs (the device's tables) == the oracle's per-pixel restatement."""
    from deva.inference.frame_io import pil_bilinear_coeffs
    for n_in, n_out in ((1, 1), (1, 9), (9, 1), (4000, 1), (97, 240), (161, 400), (480, 240), (1920, 853), (300, 299)):
        bounds, coef = pil_bilinear_coeffs(n_in, n_out)
        for o, (lo, ks) in enumerate(oracle.pil_bilinear_coeffs(n_in, n_out)):
            assert (bounds[o, 0], bounds[o, 1]) == (lo, len(ks)) and coef[o, :len(ks)].tolist() == ks, (n_in, n_out, o)
            assert not coef[o, len(ks):].any()


def test_oracle_rgb_ids_equal_pillow():
    """oracle.rgb_ids_nearest == Resize(NEAREST) of an RGB image, then r + 256 g + 65536 b."""
    rng = np.random.default_rng(5)
    for h, w, oh, ow in ((37, 53, 20, 30), (37, 53, 80, 100), (96, 160, 480, 800), (17, 9, 853, 480), (5, 5, 5, 5)):
        rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        m = np.array(Image.fromarray(rgb).resize((ow, oh), Image.NEAREST), dtype=np.int32)
        np.testing.assert_array_equal(oracle.rgb_ids_nearest(rgb, oh, ow),
                                      m[:, :, 0] + m[:, :, 1] * 256 + m[:, :, 2] * 256 * 256)


def test_readers_import_without_pycocotools_or_cuda():
    """The readers and the loader import with pycocotools unavailable and leave CUDA uninitialised."""
    code = textwrap.dedent("""
        import sys
        sys.modules['pycocotools'] = None
        import torch
        import deva.inference.data.video_reader, deva.inference.data.detection_video_reader
        import deva.inference.data.device_loader
        print(torch.cuda.is_initialized())
    """)
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True,
                         env=dict(os.environ, PYTHONPATH=PKG + os.pathsep + ROOT))
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == 'False'


def test_reference_datasets_yield_our_reader(tmp_path):
    """With this package first on sys.path and a reference checkout after it, the checkout's dataset listings import
    our ``VideoReader``."""
    data = tmp_path / 'deva' / 'inference' / 'data'
    data.mkdir(parents=True)
    for d in (tmp_path / 'deva', tmp_path / 'deva' / 'inference', data):
        (d / '__init__.py').write_text('')
    (data / 'vos_test_datasets.py').write_text('from deva.inference.data.video_reader import VideoReader\n')
    (data / 'video_reader.py').write_text('raise RuntimeError("the reference reader must not load")\n')
    code = 'import deva.inference.data.vos_test_datasets as v; print(v.VideoReader.__module__, v.__file__)'
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True,
                         env=dict(os.environ, PYTHONPATH=PKG + os.pathsep + str(tmp_path)))
    assert out.returncode == 0, out.stderr
    module, listing = out.stdout.split()
    assert module == 'deva.inference.data.video_reader' and listing.startswith(str(tmp_path))
