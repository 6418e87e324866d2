"""PNG files of the decoder tests (tests/test_png_decode_cpu.py against Pillow and oracle/png_decode.py,
tests/test_png_decode_gpu.py against Pillow), regenerated from fixed seeds: ``cases(large)`` -> [(case id, file bytes)].

Writers: Pillow at every compress level and optimize=True; OpenCV at several levels, every strategy and each single
filter; a hand-built writer (``build``) that forces a filter type per row and drives zlib with every strategy, small
windows, stored blocks over 64 KiB and IDAT splits at odd boundaries; this project's device PNG encoder (restated byte
for byte by oracle/png_encode.py).  Content: ellipse id maps, noise and gradients, every eligible mode and depth with
widths that end mid-byte, 1x1 to 4K.  Fixtures: the DAVIS bmx-trees annotation and four VIPSeg detection maps of the
project's examples.  Malformed files (``malformed``): Pillow's tolerated quirks, every class of zlib error the device
checks, truncated files, bad CRCs and the modes the device leaves to Pillow."""
import io
import os
import struct
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = ['png_decode_davis_bmx-trees_00000.png'] + [f'png_decode_vipseg_{n:08d}.png' for n in (1255, 1258, 1261,
                                                                                                    1264)]
SIG = b'\x89PNG\r\n\x1a\n'
COLOUR = {'L': 0, 'RGB': 2, 'P': 3, 'RGBA': 6}
CHANNELS = {'L': 1, 'RGB': 3, 'P': 1, 'RGBA': 4}


def chunk(kind: bytes, data: bytes, crc=None) -> bytes:
    crc = zlib.crc32(kind + data) if crc is None else crc
    return struct.pack('>I', len(data)) + kind + data + struct.pack('>I', crc)


def ellipses(h, w, k=16, seed=0):
    rng = np.random.default_rng(seed)
    ids = np.zeros((h, w), np.int32)
    yy, xx = np.ogrid[:h, :w]
    for i in range(1, k + 1):
        cy, cx = rng.uniform(0, h), rng.uniform(0, w)
        ry, rx = rng.uniform(h / 20, h / 4) + 0.5, rng.uniform(w / 20, w / 4) + 0.5
        ids[((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1] = i
    return ids


def image(content, mode, h, w, seed=0, levels=256):
    """uint8 [h, w] or [h, w, c] of 'ellipse', 'noise' or 'gradient' content with values below ``levels``."""
    rng = np.random.default_rng(seed)
    c = CHANNELS[mode]
    if content == 'ellipse':
        ids = ellipses(h, w, 16 if levels > 16 else max(levels - 1, 1), seed)
        lut = rng.integers(0, levels, (64, c), dtype=np.int64)
        img = lut[ids % 64]
    elif content == 'noise':
        img = rng.integers(0, levels, (h, w, c))
    else:
        yy, xx = np.mgrid[:h, :w]
        img = np.stack([(yy * (3 + k) + xx * (5 + 2 * k)) % levels for k in range(c)], -1)
    img = img.astype(np.uint8)
    return np.ascontiguousarray(img[:, :, 0] if c == 1 else img)


def pillow(img, mode, bits=8, **kw):
    from PIL import Image
    im = Image.fromarray(img, 'L' if mode == 'P' else mode)
    if mode == 'P':
        im = Image.frombytes('P', (img.shape[1], img.shape[0]), img.tobytes())
        im.putpalette(bytes((37 * i + 11) % 256 for i in range(3 * (1 << bits))))
    buf = io.BytesIO()
    im.save(buf, 'PNG', **kw)
    return buf.getvalue()


def paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def pack(img, mode, bits):
    """Rows of raw PNG bytes [h, rowbytes] of an image ([h, w] values < 2^bits, or [h, w, c] at 8 bits)."""
    h = img.shape[0]
    if bits == 8:
        return img.reshape(h, -1).astype(np.int32)
    return np.packbits(np.unpackbits(img[:, :, None], axis=2)[:, :, 8 - bits:].reshape(h, -1), axis=1).astype(np.int32)


def filtered(raw, bpp, filters):
    """The filtered stream of rows ``raw`` [h, rowbytes] with filter type filters[y] on row y (types 0-4)."""
    h, n = raw.shape
    up = np.vstack([np.zeros((1, n), np.int32), raw[:-1]])
    left = np.hstack([np.zeros((h, bpp), np.int32), raw[:, :-bpp]]) if n > bpp else np.zeros_like(raw)
    ul = np.hstack([np.zeros((h, bpp), np.int32), up[:, :-bpp]]) if n > bpp else np.zeros_like(raw)
    preds = [np.zeros_like(raw), left, up, (left + up) >> 1, paeth(left, up, ul)]
    out = np.empty((h, n + 1), np.uint8)
    for y in range(h):
        f = filters[y] % 5
        out[y, 0] = filters[y]
        out[y, 1:] = (raw[y] - preds[f][y]) & 255
    return out.tobytes()


def build(img, mode, bits=8, filters=None, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=15, split=None,
          before=(), after=(), stream=None, palette_entries=None, interlace=0, colour=None):
    """A PNG file written here: per-row filter types (an int for all rows, a list, or None for a seeded mix), zlib's
    settings, IDAT split at the given sizes, extra chunks (kind, data) before and after the IDATs; ``stream`` replaces
    the zlib stream (for malformed streams)."""
    h, w = img.shape[:2]
    c = CHANNELS[mode]
    raw = pack(img, mode, bits)
    bpp = max(1, c * bits // 8)
    if filters is None:
        filters = list(np.random.default_rng(h * 7 + w).integers(0, 5, h))
    elif isinstance(filters, int):
        filters = [filters] * h
    s = filtered(raw, bpp, filters)
    if stream is None:
        co = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
        stream = co.compress(s) + co.flush()
    elif callable(stream):
        stream = stream(s)
    out = SIG + chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, bits, COLOUR[mode] if colour is None else colour, 0, 0,
                                           interlace))
    if mode == 'P':
        n = palette_entries or (1 << bits)
        out += chunk(b'PLTE', bytes((53 * i + 7) % 256 for i in range(3 * n)))
    for kind, data in before:
        out += chunk(kind, data)
    parts, at = [], 0
    for n in (split or []):
        parts.append(stream[at:at + n])
        at += n
    parts.append(stream[at:])
    for p in parts:
        out += chunk(b'IDAT', p)
    for kind, data in after:
        out += chunk(kind, data)
    return out + chunk(b'IEND', b'')


def levels_of(mode, bits):
    return 1 << bits if mode in ('L', 'P') else 256


def opencv(img, mode, params):
    import cv2
    a = img[:, :, ::-1] if mode in ('RGB', 'RGBA') else img
    if mode == 'RGBA':
        a = np.ascontiguousarray(img[:, :, [2, 1, 0, 3]])
    ok, buf = cv2.imencode('.png', np.ascontiguousarray(a), params)
    assert ok
    return buf.tobytes()


def device_encoder(img, mode, bits=8):
    from oracle import png_encode as op
    palette = [(37 * i + 11) % 256 for i in range(3 * (1 << bits))] if mode == 'P' else None
    return op.encode_png(img, mode, palette)


ANCILLARY = [(b'tRNS', None), (b'gAMA', struct.pack('>I', 45455)), (b'cHRM', bytes(range(32))), (b'sRGB', b'\x00'),
             (b'pHYs', struct.pack('>IIB', 2835, 2835, 1)), (b'sBIT', None), (b'bKGD', None),
             (b'tEXt', b'Comment\x00written by the tests'), (b'tIME', struct.pack('>HBBBBB', 2024, 5, 6, 7, 8, 9))]


def ancillary_data(kind, data, mode):
    if data is not None:
        return data
    if kind == b'tRNS':
        return {'L': b'\x00\x07', 'RGB': b'\x00\x01\x00\x02\x00\x03', 'P': b'\x00\x80\xff'}[mode]
    if kind == b'sBIT':
        return bytes([8] * {'L': 1, 'P': 3, 'RGB': 3, 'RGBA': 4}[mode])
    return {'L': b'\x00\x05', 'P': b'\x02', 'RGB': b'\x00\x01\x00\x02\x00\x03', 'RGBA': b'\x00\x01\x00\x02\x00\x03'}[mode]


def valid_cases(large=False):
    """[(id, bytes)] of well-formed files."""
    out = []
    small = [(1, 1), (1, 37), (29, 1), (13, 7), (37, 53), (64, 96)]
    # Pillow: every compress level and optimize, on id maps in every mode it writes at 8 bits
    for mode in ('L', 'RGB', 'RGBA', 'P'):
        img = image('ellipse', mode, 45, 67)
        for lvl in range(10):
            out.append((f'pil-{mode}-l{lvl}-45x67', pillow(img, mode, compress_level=lvl)))
        out.append((f'pil-{mode}-opt-45x67', pillow(img, mode, optimize=True)))
    for mode, bits in (('P', 1), ('P', 2), ('P', 4)):
        for h, w in small:
            out.append((f'pil-P{bits}-ellipse-{h}x{w}', pillow(image('ellipse', mode, h, w, levels=1 << bits), mode,
                                                               bits)))
    # OpenCV: levels, strategies, single filters
    import cv2
    for mode in ('L', 'RGB', 'RGBA'):
        img = image('ellipse', mode, 50, 70, seed=3)
        for lvl in (0, 1, 3, 6, 9):
            out.append((f'cv-{mode}-l{lvl}', opencv(img, mode, [cv2.IMWRITE_PNG_COMPRESSION, lvl])))
        for name in ('DEFAULT', 'FILTERED', 'HUFFMAN_ONLY', 'RLE', 'FIXED'):
            out.append((f'cv-{mode}-{name}', opencv(img, mode, [cv2.IMWRITE_PNG_STRATEGY,
                                                                getattr(cv2, f'IMWRITE_PNG_STRATEGY_{name}')])))
        for name in ('NONE', 'SUB', 'UP', 'AVG', 'PAETH'):
            out.append((f'cv-{mode}-filter-{name}', opencv(img, mode, [cv2.IMWRITE_PNG_FILTER,
                                                                       getattr(cv2, f'IMWRITE_PNG_FILTER_{name}')])))
    # hand-built: each filter on every row, mixed filters, every mode and depth at widths that end mid-byte
    for mode, bits in (('L', 2), ('L', 4), ('L', 8), ('P', 1), ('P', 2), ('P', 4), ('P', 8), ('RGB', 8), ('RGBA', 8)):
        for content in ('ellipse', 'noise', 'gradient'):
            for h, w in ((1, 1), (3, 5), (17, 13), (31, 19), (40, 61)):
                img = image(content, mode, h, w, seed=h + w, levels=levels_of(mode, bits))
                for f in (0, 1, 2, 3, 4, None):
                    out.append((f'hand-{mode}{bits}-{content}-{h}x{w}-f{"mix" if f is None else f}',
                                build(img, mode, bits, f)))
    # zlib settings, stored blocks over 64 KiB, IDAT splits
    img = image('ellipse', 'RGB', 96, 128, seed=5)
    for name in ('Z_DEFAULT_STRATEGY', 'Z_FILTERED', 'Z_HUFFMAN_ONLY', 'Z_RLE', 'Z_FIXED'):
        for wbits in (9, 10, 12, 15):
            out.append((f'zlib-{name}-w{wbits}', build(img, 'RGB', strategy=getattr(zlib, name), wbits=wbits)))
    big = image('noise', 'RGB', 200, 150, seed=6)
    out.append(('zlib-stored-200x150', build(big, 'RGB', level=0)))
    out.append(('zlib-stored-split', build(big, 'RGB', level=0, split=[1, 7, 65535, 3, 40000])))
    out.append(('idat-split-1', build(img, 'RGB', split=[1] * 50)))
    out.append(('idat-split-odd', build(img, 'RGB', split=[3, 5, 7, 11, 13, 17, 19, 23, 29, 31])))
    out.append(('idat-empty-chunks', build(img, 'RGB', split=[0, 10, 0, 0, 5])))
    # this project's device encoder (fixed codes, Up rows)
    for mode, bits in (('L', 8), ('RGB', 8), ('P', 1), ('P', 2), ('P', 4), ('P', 8)):
        for h, w in small:
            out.append((f'dev-{mode}{bits}-{h}x{w}', device_encoder(image('ellipse', mode, h, w, levels=1 << bits
                                                                          if mode == 'P' else 256), mode, bits)))
    # allowlisted ancillary chunks
    for mode in ('L', 'RGB', 'RGBA', 'P'):
        img = image('ellipse', mode, 21, 33, levels=256 if mode != 'P' else 16)
        bits = 4 if mode == 'P' else 8
        for kind, data in ANCILLARY:
            if kind == b'tRNS' and mode == 'RGBA':
                continue
            d = ancillary_data(kind, data, mode)
            out.append((f'anc-{mode}-{kind.decode()}', build(img, mode, bits, before=[(kind, d)])))
        out.append((f'anc-{mode}-after', build(img, mode, bits, after=[(b'tEXt', b'k\x00v'), (b'tIME', ANCILLARY[-1][1])])))
    # fixtures
    for name in FIXTURES:
        with open(os.path.join(HERE, name), 'rb') as f:
            out.append((f'fixture-{name}', f.read()))
    # sizes
    out.append(('pil-RGB-ellipse-480x854', pillow(image('ellipse', 'RGB', 480, 854), 'RGB')))
    out.append(('pil-P-ellipse-480x854', pillow(image('ellipse', 'P', 480, 854), 'P')))
    if large:
        for h, w in ((720, 1280), (1080, 1920), (2160, 3840)):
            out.append((f'pil-RGB-ellipse-{h}x{w}', pillow(image('ellipse', 'RGB', h, w), 'RGB')))
            out.append((f'pil-L-gradient-{h}x{w}', pillow(image('gradient', 'L', h, w), 'L')))
        out.append(('pil-RGB-noise-1080x1920', pillow(image('noise', 'RGB', 1080, 1920), 'RGB')))
        out.append(('dev-RGB-ellipse-1080x1920', device_encoder(image('ellipse', 'RGB', 1080, 1920), 'RGB')))
        out.append(('hand-RGBA-mix-720x1280', build(image('ellipse', 'RGBA', 720, 1280), 'RGBA')))
    return out


# ---------------------------------------------------------------------------------------------- malformed streams
class BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, v, n):  # LSB first
        self.bits += [(v >> i) & 1 for i in range(n)]

    def code(self, c, n):  # Huffman codes MSB first
        self.bits += [(c >> (n - 1 - i)) & 1 for i in range(n)]

    def align(self):
        self.bits += [0] * (-len(self.bits) % 8)

    def bytes(self):
        self.align()
        return bytes(int(''.join(map(str, self.bits[i:i + 8][::-1])), 2) for i in range(0, len(self.bits), 8))


def fixed_literal(bw, v):
    if v < 144:
        bw.code(0x30 + v, 8)
    else:
        bw.code(0x190 + v - 144, 9)


def fixed_symbol(bw, sym):
    if sym < 256:
        fixed_literal(bw, sym)
    elif sym < 280:
        bw.code(sym - 256, 7)
    else:
        bw.code(0xC0 + sym - 280, 8)


def zlib_wrap(body: bytes, s: bytes, header=b'\x78\x01') -> bytes:
    return header + body + struct.pack('>I', zlib.adler32(s))


def fixed_stream(s, tail=None):
    """s as fixed-code literals, then the symbols ``tail`` (list of ('sym', v) / ('bits', v, n)), end-of-block."""
    bw = BitWriter()
    bw.put(1, 1)
    bw.put(1, 2)
    for v in s:
        fixed_literal(bw, v)
    for t in tail or []:
        if t[0] == 'sym':
            fixed_symbol(bw, t[1])
        else:
            bw.put(t[1], t[2])
    fixed_symbol(bw, 256)
    return bw.bytes()


def dynamic_header(bw, clen_lengths, hlit=257, hdist=1):
    bw.put(1, 1)
    bw.put(2, 2)
    bw.put(hlit - 257, 5)
    bw.put(hdist - 1, 5)
    bw.put(len(clen_lengths) - 4, 4)
    for v in clen_lengths:
        bw.put(v, 3)


def malformed():
    """[(id, bytes)]: files the device must not accept (or, for the ineligible ones, not even see)."""
    img = image('ellipse', 'L', 9, 11, seed=9)
    raw = pack(img, 'L', 8)
    s = filtered(raw, 1, [0] * 9)
    good = zlib.compress(s)
    out = []

    def with_stream(name, stream):
        out.append((name, build(img, 'L', stream=stream)))

    # Pillow's quirks
    f = build(img, 'L')
    crc = f.index(b'IEND') - 8  # the IDAT's CRC ends where IEND's length begins
    out.append(('quirk-bad-idat-crc', f[:crc] + bytes([f[crc] ^ 0xff]) + f[crc + 1:]))
    with_stream('quirk-stream-ends-early', good[:len(good) // 2])
    with_stream('quirk-trailing-bytes', good + b'\x00junk')
    with_stream('quirk-extra-inflated', zlib.compress(s + b'\x00' * 12))
    with_stream('quirk-bad-adler', good[:-4] + bytes([good[-4] ^ 1]) + good[-3:])
    bad_filter = bytearray(s)
    bad_filter[12 * 3] = 5
    with_stream('quirk-filter-5', zlib.compress(bytes(bad_filter)))
    bad_filter[12 * 3] = 200
    with_stream('quirk-filter-200', zlib.compress(bytes(bad_filter)))
    # zlib header
    with_stream('hdr-bad-check', b'\x78\x02' + good[2:])
    with_stream('hdr-method-7', b'\x77' + good[1:])
    with_stream('hdr-window-64k', b'\x88\x1c' + good[2:])
    with_stream('hdr-fdict', b'\x78\x20' + b'\x00\x00\x00\x01' + good[2:])
    # blocks
    with_stream('blk-type-3', zlib_wrap(bytes([0b111]) + b'\x00' * 8, s))
    stored = b'\x01' + struct.pack('<HH', len(s), 0xffff ^ len(s) ^ 1) + s
    with_stream('blk-stored-nlen', zlib_wrap(stored, s))
    bw = BitWriter()
    dynamic_header(bw, [1] * 19)
    with_stream('blk-oversubscribed', zlib_wrap(bw.bytes() + b'\x00' * 16, s))
    bw = BitWriter()
    dynamic_header(bw, [0, 0, 0, 2])  # one code-length code of 2 bits: incomplete
    with_stream('blk-incomplete-clen', zlib_wrap(bw.bytes() + b'\x00' * 16, s))
    # incomplete literal/length code: code-length code all 4-bit (16 codes among 19... complete set of 16 at length 4)
    bw = BitWriter()
    clen = [0] * 19
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    for sym in range(16):
        clen[order.index(sym)] = 4
    dynamic_header(bw, clen)
    for sym in range(258):  # literal/length lengths: every one 9 bits (257 of 512: incomplete), one distance of 1
        bw.code(9 if sym < 257 else 1, 4)
    with_stream('blk-incomplete-litlen', zlib_wrap(bw.bytes() + b'\x00' * 16, s))
    with_stream('sym-286', zlib_wrap(fixed_stream(s[:5], [('sym', 286)]), s))
    with_stream('sym-287', zlib_wrap(fixed_stream(s[:5], [('sym', 287)]), s))
    with_stream('dist-30', zlib_wrap(fixed_stream(s[:5], [('sym', 257), ('bits', 0b01111, 5)]), s))
    with_stream('dist-31', zlib_wrap(fixed_stream(s[:5], [('sym', 257), ('bits', 0b11111, 5)]), s))
    with_stream('dist-before-start', zlib_wrap(fixed_stream(s[:2], [('sym', 257), ('bits', 0b00100, 5)]), s))
    with_stream('stream-too-short', zlib.compress(s[:-3]))
    with_stream('stream-too-long', zlib.compress(s + b'\x00'))
    with_stream('stream-empty', b'')
    with_stream('stream-two', good + good)
    # files
    full = build(img, 'L')
    for n in (7, 20, 40, len(full) // 2, len(full) - 13, len(full) - 1):
        out.append((f'file-truncated-{n}', full[:n]))
    ihdr = full.index(b'IHDR')
    out.append(('file-bad-ihdr-crc', full[:ihdr + 17] + bytes([full[ihdr + 17] ^ 1]) + full[ihdr + 18:]))
    out.append(('file-bad-text-crc', build(img, 'L', before=[(b'tEXt', b'a\x00b')]).replace(
        chunk(b'tEXt', b'a\x00b'), chunk(b'tEXt', b'a\x00b', crc=1))))
    out.append(('file-after-iend', full + b'\x00'))
    out.append(('file-not-png', b'GIF89a' + full[6:]))
    out.append(('file-unknown-chunk', build(img, 'L', before=[(b'zzZz', b'x')])))
    out.append(('file-short-phys', build(img, 'L', before=[(b'pHYs', b'\x00' * 4)])))
    # modes the device leaves to Pillow
    bits1 = image('noise', 'L', 7, 13, levels=2)
    out.append(('mode-1bit-grey', build(bits1, 'L', 1)))
    la = image('noise', 'RGB', 6, 5)[:, :, :2]
    out.append(('mode-LA', SIG + chunk(b'IHDR', struct.pack('>IIBBBBB', 5, 6, 8, 4, 0, 0, 0)) +
                chunk(b'IDAT', zlib.compress(filtered(la.reshape(6, -1).astype(np.int32), 2, [0] * 6))) +
                chunk(b'IEND', b'')))
    g16 = image('noise', 'L', 5, 4).astype(np.uint16) * 257
    out.append(('mode-L16', SIG + chunk(b'IHDR', struct.pack('>IIBBBBB', 4, 5, 16, 0, 0, 0, 0)) +
                chunk(b'IDAT', zlib.compress(filtered(g16.astype('>u2').view(np.uint8).reshape(5, -1).astype(np.int32),
                                                      2, [0] * 5))) + chunk(b'IEND', b'')))
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(image('ellipse', 'RGB', 16, 16)).save(buf, 'PNG', save_all=True, append_images=[
        Image.fromarray(image('noise', 'RGB', 16, 16))])
    out.append(('mode-apng', buf.getvalue()))
    out.append(('mode-adam7', build(image('ellipse', 'L', 8, 8), 'L', interlace=1)))
    out.append(('mode-no-plte', build(image('ellipse', 'L', 8, 8), 'L', colour=3)))
    return out


def cases(large=False):
    return valid_cases(large) + malformed()
