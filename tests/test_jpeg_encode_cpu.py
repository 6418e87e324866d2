"""The baseline JPEG of deva/utils/jpeg_encode.py, restated on the CPU by oracle/jpeg_encode.py: its files are byte for
byte Pillow's ``Image.fromarray(img).save(f, 'JPEG')`` (and ``quality=q``) over shapes from 1x1 to 1080p, every h and w
residue mod 16, constant, gradient, noise, saturated and overlay content, qualities 1 to 100, and scans whose 1-bit
fill makes a 0xFF byte.  Also the package's tables and markers, its encoder option and input checks.  No GPU."""
import io
import os
import subprocess
import sys

import numpy as np
import pytest
from PIL import Image

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import jpeg_cases as jc  # noqa: E402

from oracle import jpeg_encode as oj  # noqa: E402


def pillow_jpeg(img, quality):
    buf = io.BytesIO()
    if quality == 75:
        Image.fromarray(img).save(buf, 'JPEG')  # Pillow's default
    else:
        Image.fromarray(img).save(buf, 'JPEG', quality=quality)
    return buf.getvalue()


@pytest.mark.parametrize('case', jc.case_ids(large=False))
def test_oracle_matches_pillow(case):
    img, q = jc.make(case)
    assert oj.encode_jpeg(img, q) == pillow_jpeg(img, q), case


@pytest.mark.parametrize('case', jc.case_ids(large=True))
def test_oracle_matches_pillow_large(case):
    test_oracle_matches_pillow(case)


def test_cases_cover_every_residue():
    shapes = [tuple(int(v) for v in c.split('-')[1].split('x')) for c in jc.case_ids(large=False)]
    assert {h % 16 for h, _ in shapes} == set(range(16))
    assert {w % 16 for _, w in shapes} == set(range(16))


@pytest.mark.parametrize('case', jc.FILL_FF)
def test_fill_byte_0xff_is_stuffed(case):
    """The last scan byte is the 1-bit fill's 0xFF, followed by its stuffed 0x00 and EOI."""
    img, q = jc.make(case)
    coef, comp = oj.coefficients(img, q)
    _, lens = oj._tokens(coef, comp)
    assert lens.sum() % 8 != 0
    data = oj.encode_jpeg(img, q)
    assert data.endswith(b'\xff\x00\xff\xd9')
    assert data == pillow_jpeg(img, q)


def test_noise_scan_stuffs_0xff():
    img, q = jc.make('noise-120x200-q75')
    data = oj.encode_jpeg(img, q)
    scan = data[len(oj.headers(120, 200, q)):-2]
    assert scan.count(b'\xff') > 10 and scan.count(b'\xff') == scan.count(b'\xff\x00')


def test_package_tables_and_markers_match_oracle():
    from deva.utils.jpeg_encode import headers, quant_tables
    for q in range(1, 101):
        lq, cq = oj.quant_tables(q)
        assert quant_tables(q) == lq.tobytes() + cq.tobytes(), q
    for h, w in [(1, 1), (37, 53), (1080, 1920), (65535, 65535)]:
        assert headers(h, w, 75) == oj.headers(h, w, 75)
    assert headers(7, 9, 1) == oj.headers(7, 9, 1)


def test_bad_inputs_raise():
    """Checked on the host, before anything reaches the device."""
    from deva.utils.jpeg_encode import encode_jpeg_async
    rgb = np.zeros((4, 5, 3), np.uint8)
    for bad in (np.zeros((4, 5), np.uint8), np.zeros((4, 5, 4), np.uint8), rgb.astype(np.int32),
                rgb.astype(np.float32), np.zeros((0, 5, 3), np.uint8), np.zeros((1, 65536, 3), np.uint8)):
        with pytest.raises(ValueError):
            encode_jpeg_async(bad)
    for q in (0, 101, -5, 75.5):
        with pytest.raises(ValueError, match='quality'):
            encode_jpeg_async(rgb, quality=q)


def test_resolve_encoder(monkeypatch):
    from deva.utils.jpeg_encode import resolve_encoder
    monkeypatch.delenv('DEVA_B200_JPEG_ENCODER', raising=False)
    assert resolve_encoder() == 'pil'
    assert resolve_encoder('device') == 'device'
    monkeypatch.setenv('DEVA_B200_JPEG_ENCODER', 'device')
    assert resolve_encoder() == 'device'
    assert resolve_encoder('pil') == 'pil'
    with pytest.raises(ValueError, match='jpeg_encoder'):
        resolve_encoder('nvjpeg')


def test_saver_reads_the_encoder_option(monkeypatch):
    from deva.inference.object_manager import ObjectManager
    from deva.inference.result_utils import ResultSaver
    monkeypatch.delenv('DEVA_B200_JPEG_ENCODER', raising=False)
    for arg, env, want in [(None, None, 'pil'), ('device', None, 'device'), (None, 'device', 'device'),
                           ('pil', 'device', 'pil')]:
        if env is not None:
            monkeypatch.setenv('DEVA_B200_JPEG_ENCODER', env)
        saver = ResultSaver('/nonexistent', None, dataset='demo', object_manager=ObjectManager(), jpeg_encoder=arg)
        assert saver.jpeg_encoder == want
        saver.end()
    with pytest.raises(ValueError, match='jpeg_encoder'):
        ResultSaver('/nonexistent', None, dataset='demo', object_manager=ObjectManager(), jpeg_encoder='nvjpeg')


def test_import_does_not_initialise_cuda():
    code = ('import torch, deva.utils.jpeg_encode, deva.inference.result_utils; '
            'assert not torch.cuda.is_initialized()')
    subprocess.run([sys.executable, '-c', code], check=True, cwd=os.path.dirname(os.path.abspath(__file__)),
                   env={**os.environ, 'PYTHONPATH': os.pathsep.join(sys.path)})
