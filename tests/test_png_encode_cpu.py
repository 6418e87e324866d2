"""The PNG format of deva/utils/png_encode.py, restated on the CPU by oracle/png_encode.py: its files are valid (zlib,
chunk CRCs) and decode in Pillow to what Pillow's own write-then-read of the same image gives - pixels, mode and
palette - for L, RGB and P images with 2 / 4 / 16 / 17 / 256-colour palettes (indices beyond the palette included),
shapes from 1x1 to 4K, constant, ellipse and noise images and rows ending in runs of 254-259 bytes; the worst-case
bound holds on noise.  Also the package's layout rule and encoder option.  No GPU."""
import io
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest
from PIL import Image

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import png_cases as pc  # noqa: E402

from oracle import png_encode as op  # noqa: E402


def _chunks(data):
    assert data[:8] == op.SIGNATURE
    out, k = [], 8
    while k < len(data):
        n, = struct.unpack('>I', data[k:k + 4])
        kind, body = data[k + 4:k + 8], data[k + 8:k + 8 + n]
        crc, = struct.unpack('>I', data[k + 8 + n:k + 12 + n])
        assert crc == zlib.crc32(kind + body), kind
        out.append((kind, body))
        k += 12 + n
    return out


def _pillow(img, mode, palette):
    im = Image.fromarray(img)
    if mode == 'P':
        im.putpalette(palette)
    buf = io.BytesIO()
    im.save(buf, format='PNG')
    back = Image.open(io.BytesIO(buf.getvalue()))
    back.load()
    return back


@pytest.mark.parametrize('case', pc.case_ids(large=False))
def test_oracle_decodes_like_pillow(case):
    img, mode, palette = pc.make(case)
    data = op.encode_png(img, mode, palette)
    chunks = _chunks(data)
    kinds = [k for k, _ in chunks]
    assert kinds == [b'IHDR'] + ([b'PLTE'] if mode == 'P' else []) + [b'IDAT', b'IEND']
    bits, plte = op.layout(mode, palette)[1:]
    h, w = img.shape[:2]
    assert chunks[0][1] == struct.pack('>IIBBBBB', w, h, bits, op.layout(mode, palette)[0], 0, 0, 0)
    idat = dict(chunks)[b'IDAT']
    s = op.filtered(img, bits)
    assert zlib.decompress(idat) == s.tobytes()
    assert len(idat) <= op.bound(h, s.shape[1] - 1)
    ours = Image.open(io.BytesIO(data))
    ours.load()
    ref = _pillow(img, mode, palette)
    assert ours.mode == ref.mode
    assert ours.getpalette() == ref.getpalette()
    np.testing.assert_array_equal(np.asarray(ours), np.asarray(ref))


@pytest.mark.parametrize('case', pc.case_ids(large=True))
def test_oracle_decodes_like_pillow_large(case):
    test_oracle_decodes_like_pillow(case)


def test_bound_holds_on_noise():
    rng = np.random.default_rng(3)
    for h, w, ch in [(1, 1, 1), (7, 13, 3), (256, 300, 1), (97, 211, 3)]:
        img = rng.integers(0, 256, (h, w, ch) if ch == 3 else (h, w), dtype=np.uint8)
        z = op.zlib_stream(img, 8, ch)
        assert len(z) <= op.bound(h, w * ch)
        assert len(z) > 0.9 * op.bound(h, w * ch)  # noise is nearly all 9-bit literals


def test_runs_at_row_end_use_length_258():
    """Constant rows of 259 bytes: the filter byte and the first byte are literals, then one 258-byte match ends at the
    row's end (row 1 is Up-filtered to zeros, the first of which follows the filter byte 2)."""
    img = np.full((2, 259), 7, np.uint8)
    lengths, dists, _ = op.tokens(op.filtered(img, 8), 1)
    assert lengths.tolist() == [1, 1, 258, 1, 1, 258]
    assert dists[lengths >= 3].tolist() == [1, 1]


def test_package_layout_matches_oracle():
    from deva.utils.png_encode import pillow_png_layout
    for mode, palette in pc.LAYOUTS:
        _, bits, plte = op.layout(mode, palette)
        assert pillow_png_layout(mode, palette) == (bits, plte), (mode, None if palette is None else len(palette))


def test_layout_examples():
    """Pillow's writer packs small palettes: a 4-colour image reads back [0, 1, 2, 3, 0, 3], a 2-colour one v != 0."""
    img = np.array([[0, 1, 2, 3, 20, 255]], np.uint8)
    for n, want in [(2, [0, 1, 1, 1, 1, 1]), (4, [0, 1, 2, 3, 0, 3]), (16, [0, 1, 2, 3, 4, 15]),
                    (17, [0, 1, 2, 3, 20, 255])]:
        back = Image.open(io.BytesIO(op.encode_png(img, 'P', list(range(3 * n)))))
        assert np.asarray(back).tolist() == [want], n
        assert len(back.getpalette()) == 3 * n


def test_resolve_encoder(monkeypatch):
    from deva.utils.png_encode import resolve_encoder
    monkeypatch.delenv('DEVA_B200_PNG_ENCODER', raising=False)
    assert resolve_encoder() == 'pil'
    assert resolve_encoder('device') == 'device'
    monkeypatch.setenv('DEVA_B200_PNG_ENCODER', 'device')
    assert resolve_encoder() == 'device'
    assert resolve_encoder('pil') == 'pil'
    with pytest.raises(ValueError, match='png_encoder'):
        resolve_encoder('nvjpeg')


def test_import_does_not_initialise_cuda():
    code = ('import torch, deva.utils.png_encode, deva.inference.result_utils; '
            'assert not torch.cuda.is_initialized()')
    subprocess.run([sys.executable, '-c', code], check=True, cwd=os.path.dirname(os.path.abspath(__file__)),
                   env={**os.environ, 'PYTHONPATH': os.pathsep.join(sys.path)})
