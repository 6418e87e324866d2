"""JPEG files of the decoder tests (tests/test_jpeg_decode_cpu.py against Pillow, oracle/jpeg_decode.py and the host
build of the device algorithm; tests/test_jpeg_decode_gpu.py against Pillow), regenerated from fixed seeds.

``valid_cases(large)`` -> [(case id, file bytes)]: Pillow's writer at qualities 1 to 100, subsampling 0, 1 and 2,
optimize on and off, restart markers every block, every MCU and every row, custom quantisation tables, sizes from 1x1
to 1080x1920 covering every h mod 16 and w mod 16, and constant, gradient, noise, saturated and overlay content
(tests/golden/jpeg_cases.py); this project's encoder (oracle/jpeg_encode.py, byte for byte the device's); the DAVIS
and VIPSeg example frames.  ``ineligible()``: files the host must leave to Pillow.  ``extreme()``: files whose
dequantised coefficients reach the IDCT's range limits.  ``mutants(files, n, seed)``: bit flips and truncations."""
import io
import os

import numpy as np

import jpeg_cases as jc

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = ['jpeg_decode_davis_bmx-trees_00000.jpg', 'jpeg_decode_vipseg_00001255.jpg']
QUALITIES = [1, 10, 50, 75, 90, 95, 100]
CONTENTS = ['const', 'gradient', 'noise', 'saturated', 'overlay']


def pillow(img, **kw) -> bytes:
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(img)).save(b, 'JPEG', **kw)
    return b.getvalue()


def image(content, h, w, seed=0):
    return np.ascontiguousarray(jc.make(f'{content}-{h}x{w}-q75')[0]) if content != 'overlay' or seed == 0 else \
        jc.overlay(h, w, seed=seed)


def fixture(name) -> bytes:
    with open(os.path.join(HERE, name), 'rb') as f:
        return f.read()


def valid_cases(large=False):
    out = []
    if large:
        for content in ('overlay', 'noise'):
            for q in (75, 95):
                for ss in (0, 2):
                    out.append((f'{content}-1080x1920-q{q}-s{ss}', pillow(image(content, 1080, 1920), quality=q,
                                                                            subsampling=ss)))
        out.append(('overlay-2160x3840-q75-s2', pillow(image('overlay', 2160, 3840), quality=75, subsampling=2)))
        out.append(('overlay-2160x3840-q95-s0', pillow(image('overlay', 2160, 3840), quality=95, subsampling=0)))
        return out
    for content in CONTENTS:
        for h, w in jc.SHAPES:
            for ss in (0, 1, 2):
                out.append((f'{content}-{h}x{w}-s{ss}', pillow(image(content, h, w), quality=75, subsampling=ss)))
    for h, w in jc.RESIDUES:
        for ss in (0, 1, 2):
            out.append((f'overlay-{h}x{w}-s{ss}', pillow(image('overlay', h, w), quality=75, subsampling=ss)))
    for q in QUALITIES:
        for content in ('overlay', 'noise', 'gradient'):
            for ss in (0, 2):
                for opt in (False, True):
                    out.append((f'{content}-37x53-q{q}-s{ss}-o{int(opt)}',
                                pillow(image(content, 37, 53), quality=q, subsampling=ss, optimize=opt)))
    img = image('overlay', 120, 200)
    for ss in (0, 1, 2):
        for k in (1, 2, 5):
            out.append((f'restart-blocks{k}-s{ss}', pillow(img, quality=80, subsampling=ss, restart_marker_blocks=k)))
        out.append((f'restart-rows1-s{ss}', pillow(img, quality=80, subsampling=ss, restart_marker_rows=1)))
    rng = np.random.default_rng(5)
    for k in range(3):
        tables = [list(rng.integers(1, 256, 64)), list(rng.integers(1, 100, 64))]
        out.append((f'qtables{k}', pillow(image('overlay', 64, 96), qtables=tables, subsampling=2)))
    out.append(('qtables-ones', pillow(image('noise', 40, 40), qtables=[[1] * 64, [1] * 64], subsampling=0)))
    out.append(('overlay-480x854-q75', pillow(jc.overlay(480, 854, seed=3), quality=75)))
    out.append(('overlay-720x1280-q95', pillow(jc.overlay(720, 1280, seed=4), quality=95)))
    from oracle import jpeg_encode
    for case in ('overlay-37x53-q75', 'noise-33x17-q95', 'gradient-120x200-q50', 'overlay-481x857-q90'):
        img, q = jc.make(case)
        out.append((f'encode_jpeg-{case}', jpeg_encode.encode_jpeg(np.ascontiguousarray(img), q)))
    out += [(name, fixture(name)) for name in FIXTURES]
    return out


def _segment(marker, body):
    return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, 'big') + body


def ineligible():
    """[(case id, file bytes)] that ``parse`` must refuse."""
    from PIL import Image
    img = image('overlay', 48, 64)
    base = pillow(img, quality=75)
    out = [('progressive', pillow(img, progressive=True)),
           ('greyscale', pillow(img[..., 0])),
           ('trailing-data', base + b'junk'),
           ('two-eoi', base + b'\xff\xd9')]
    b = io.BytesIO()
    Image.fromarray(img).convert('CMYK').save(b, 'JPEG')
    out.append(('cmyk', b.getvalue()))
    adobe = _segment(0xEE, b'Adobe\x00\x64\x00\x00\x00\x00\x00')  # transform 0: RGB
    out.append(('adobe-rgb', base[:2] + adobe + base[2:]))
    out.append(('adobe-ycc', base[:2] + _segment(0xEE, b'Adobe\x00\x64\x00\x00\x00\x00\x01') + base[2:]))
    sof = base.index(b'\xff\xc0')
    rgb_ids = bytearray(base)
    for c in range(3):
        rgb_ids[sof + 10 + 3 * c] = b'RGB'[c]
    sos = bytes(rgb_ids).index(b'\xff\xda')
    for c in range(3):
        rgb_ids[sos + 5 + 2 * c] = b'RGB'[c]
    out.append(('rgb-ids', bytes(rgb_ids)))
    b = io.BytesIO()
    Image.fromarray(img).save(b, 'MPO', save_all=True, append_images=[Image.fromarray(img[::-1].copy())])
    out.append(('mpo', b.getvalue()))
    out.append(('exif', pillow(img, exif=Image.Exif().tobytes())))
    out.append(('icc', pillow(img, icc_profile=b'\0' * 200)))
    out.append(('short-jfif', base[:2] + _segment(0xE0, b'JFIF\0\1') + base[2:]))
    out.append(('truncated-header', base[:100]))
    out.append(('no-soi', base[2:]))
    twelve = bytearray(base)
    twelve[sof + 4] = 12
    out.append(('12-bit', bytes(twelve)))
    s = pillow(image('overlay', 48, 64), quality=75, subsampling=1)
    sof = s.index(b'\xff\xc0')
    odd = bytearray(s)
    odd[sof + 11] = 0x12  # Y 1x2
    out.append(('sampling-1x2', bytes(odd)))
    return out


def extreme():
    """Files whose dequantised coefficients are as large as a baseline stream allows: Pillow's quality-100 noise and
    saturated streams (coefficients of every magnitude) with their quantisation tables replaced by large constants, so
    the dequantised values and the IDCT's intermediate sums cross the ranges where libjpeg-turbo's C and SIMD islow
    paths agree.  Each must either equal Pillow or be refused by the device."""
    out = []
    for content in ('noise', 'saturated', 'overlay'):
        for ss in (0, 2):
            f = pillow(image(content, 32, 48), quality=100, subsampling=ss)
            for qv in (2, 8, 16, 17, 32, 64, 255):
                g = bytearray(f)
                at = 0
                while True:
                    at = g.find(b'\xff\xdb', at + 1)
                    if at < 0:
                        break
                    n = int.from_bytes(g[at + 2:at + 4], 'big') - 2
                    p = at + 4
                    while p < at + 4 + n:
                        g[p + 1:p + 65] = bytes([qv]) * 64
                        p += 65
                out.append((f'extreme-{content}-s{ss}-q{qv}', bytes(g)))
    return out


def mutants(files, n, seed=0):
    """n files derived from ``files`` by flipping 1 to 3 random bits of the scan or truncating it."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        f = bytearray(files[k % len(files)])
        sos = f.index(b'\xff\xda')
        lo, hi = sos + 14, len(f) - 2
        if k % 5 == 4:
            cut = int(rng.integers(lo, hi))
            g = bytes(f[:cut]) + b'\xff\xd9'
        else:
            for _ in range(int(rng.integers(1, 4))):
                i = int(rng.integers(lo, hi))
                f[i] ^= 1 << int(rng.integers(0, 8))
            g = bytes(f)
        out.append((f'mutant{k}', g))
    return out
