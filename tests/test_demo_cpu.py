"""CPU: the demos' drop-ins (deva/inference/data/simple_video_reader.py, deva/inference/demo_utils.py) against the
fixture minted from the unmodified reference (tests/golden/demo.{json,npz}), their imports, and their input checks."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'tracking-anything-with-deva_b200')
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
REFERENCE = os.environ.get('DEVA_REFERENCE_ROOT', '/root/reference')


@pytest.fixture(scope='module')
def sc():
    sys.path.insert(0, GOLDEN)
    try:
        import demo_scenario
    finally:
        sys.path.remove(GOLDEN)
    return demo_scenario


@pytest.fixture(scope='module')
def meta():
    return json.load(open(os.path.join(GOLDEN, 'demo.json')))


@pytest.mark.parametrize('folder', ['reader', 'clip'])
def test_simple_video_reader_matches_reference(sc, meta, folder, tmp_path):
    """Names, order, every array's SHA-256 and shape, and Pillow's error at the same index."""
    from deva.inference.data.simple_video_reader import SimpleVideoReader, no_collate
    root = str(tmp_path / folder)
    (sc.write_reader_folder if folder == 'reader' else sc.write_demo_clip)(root)
    reader = SimpleVideoReader(root)
    assert len(reader) == len(meta['reader'][folder])
    assert sc.read_items(reader, root) == meta['reader'][folder]
    assert [reader.plan(i).image for i in range(len(reader))] == [os.path.join(root, f) for f in reader.frames]
    item = reader[0]
    assert no_collate(item) is item


def _run(code, *paths):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(paths))
    out = subprocess.run([sys.executable, '-c', code], env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


def test_demo_modules_import_without_cuda_or_deva_dataset():
    _run("import sys\n"
         "import torch\n"
         "import deva.inference.demo_utils as d, deva.inference.data.simple_video_reader as r\n"
         "import deva.inference.data.device_loader\n"
         f"assert d.__file__.startswith({PKG!r}) and r.__file__.startswith({PKG!r})\n"
         "assert callable(d.get_input_frame_for_deva) and callable(d.flush_buffer)\n"
         "assert 'deva.dataset' not in sys.modules\n"
         "assert not torch.cuda.is_initialized()\n", PKG)


@pytest.mark.parametrize('bad', [
    [[[0, 0, 0]]], 'frame.jpg', None,
    np.zeros((4, 5, 3), np.float32), np.zeros((4, 5), np.uint8), np.zeros((4, 5, 4), np.uint8),
    torch.zeros(4, 5, 3, dtype=torch.uint8),
])
def test_get_input_frame_rejects_other_inputs(bad):
    from deva.inference.demo_utils import get_input_frame_for_deva
    with pytest.raises(TypeError, match='get_input_frame_for_deva'):
        get_input_frame_for_deva(bad, 120)


def test_device_loader_rejects_other_readers():
    from deva.inference.data.device_loader import DeviceLoader
    with pytest.raises(TypeError, match='SimpleVideoReader, not list'):
        DeviceLoader([np.zeros((2, 2, 3), np.uint8)])


@pytest.mark.skipif(not os.path.isdir(os.path.join(REFERENCE, 'deva', 'ext')), reason='no reference checkout')
def test_reference_processors_take_demo_utils_from_this_package():
    """With this package first on sys.path, the reference's processors take get_input_frame_for_deva (and the demos
    flush_buffer and SimpleVideoReader) from here, and still come from the checkout themselves."""
    _run("import sys, types\n"
         "for name in ('segment_anything', 'groundingdino', 'groundingdino.util', 'groundingdino.util.inference'):\n"
         "    m = sys.modules[name] = types.ModuleType(name); m.__path__ = []\n"
         "    m.SamAutomaticMaskGenerator = m.SamPredictor = m.Model = object\n"
         "sys.modules['pulp'] = types.ModuleType('pulp')\n"
         "import deva.ext.automatic_processor as ap, deva.ext.with_text_processor as tp\n"
         "import deva.inference.demo_utils as du, deva.inference.data.simple_video_reader as sv\n"
         f"assert ap.get_input_frame_for_deva.__code__.co_filename.startswith({PKG!r})\n"
         f"assert tp.get_input_frame_for_deva.__code__.co_filename.startswith({PKG!r})\n"
         f"assert du.__file__.startswith({PKG!r}) and sv.__file__.startswith({PKG!r})\n"
         f"assert ap.__file__.startswith({REFERENCE!r}) and tp.__file__.startswith({REFERENCE!r})\n", PKG, REFERENCE)
