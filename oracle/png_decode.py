"""Restatement of the device PNG decoder (deva/utils/png_decode.py, csrc/png_decode.cu) in numpy: which files the host
sends to the device (``eligible``), which of them the device accepts (``accepts``), and the array it gives
(``decode``).  Inflate is zlib's; the chunk rule, unfiltering and unpacking are written out again here, so that
tests/test_png_decode_cpu.py can pin them to Pillow and tests/test_png_decode_gpu.py the device to them."""
import struct
import zlib

import numpy as np

SIGNATURE = b'\x89PNG\r\n\x1a\n'
MODES = {(0, 2): 'L', (0, 4): 'L', (0, 8): 'L', (3, 1): 'P', (3, 2): 'P', (3, 4): 'P', (3, 8): 'P', (2, 8): 'RGB',
         (6, 8): 'RGBA'}
CHANNELS = {'L': 1, 'P': 1, 'RGB': 3, 'RGBA': 4}
FIXED_LENGTHS = {b'gAMA': 4, b'cHRM': 32, b'sRGB': 1, b'pHYs': 9, b'tIME': 7}
PER_MODE_LENGTHS = {b'sBIT': {'L': 1, 'P': 3, 'RGB': 3, 'RGBA': 4}, b'bKGD': {'L': 2, 'P': 1, 'RGB': 6, 'RGBA': 6}}
MAX_PIXELS = 89478485  # Pillow's default Image.MAX_IMAGE_PIXELS
TEXT_BYTES = 1 << 20


def _chunks(data):
    """[(kind, payload)] when the file is the signature and CRC-valid chunks ending with IEND and nothing after."""
    if data[:8] != SIGNATURE:
        return None
    out, pos = [], 8
    while pos < len(data):
        if pos + 12 > len(data):
            return None
        n, kind = struct.unpack('>I4s', data[pos:pos + 8])
        payload = data[pos + 8:pos + 8 + n]
        if n >= 1 << 31 or pos + 12 + n > len(data) or \
                zlib.crc32(kind + payload) != struct.unpack('>I', data[pos + 8 + n:pos + 12 + n])[0]:
            return None
        out.append((kind, payload))
        pos += 12 + n
        if kind == b'IEND':
            return out if pos == len(data) else None
    return None


def eligible(data, max_pixels=MAX_PIXELS):
    """(h, w, colour type, bit depth, mode, zlib stream) of a device-eligible file, else None."""
    chunks = _chunks(bytes(data))
    if not chunks or len(chunks) < 3 or chunks[0][0] != b'IHDR' or len(chunks[0][1]) != 13 or chunks[-1] != (b'IEND',
                                                                                                             b''):
        return None
    w, h, bits, ct, comp, filt, lace = struct.unpack('>IIBBBBB', chunks[0][1])
    mode = MODES.get((ct, bits))
    if mode is None or comp or filt or lace or not (0 < w < 2 ** 31 and 0 < h < 2 ** 31) or w * h > max_pixels:
        return None
    kinds = [k for k, _ in chunks]
    idat = [i for i, k in enumerate(kinds) if k == b'IDAT']
    if not idat or idat[-1] - idat[0] + 1 != len(idat):
        return None
    first, last = idat[0], idat[-1]
    entries, text = 0, 0
    for i, (kind, payload) in enumerate(chunks[1:-1], 1):
        if kind == b'IDAT':
            continue
        if kinds.count(kind) > 1 and kind != b'tEXt':
            return None
        if kind == b'PLTE':
            if mode != 'P' or i > first or len(payload) % 3 or not 1 <= len(payload) // 3 <= 256:
                return None
            entries = len(payload) // 3
            continue
        if i > last and kind not in (b'tEXt', b'tIME'):
            return None
        n = len(payload)
        if kind in FIXED_LENGTHS:
            ok = n == FIXED_LENGTHS[kind]
        elif kind in PER_MODE_LENGTHS:
            ok = n == PER_MODE_LENGTHS[kind][mode]
        elif kind == b'tRNS':
            ok = (mode == 'P' and 1 <= n <= entries) or (mode == 'L' and n == 2) or (mode == 'RGB' and n == 6)
        elif kind == b'tEXt':
            ok = True
            text += n
        else:
            ok = False
        if not ok:
            return None
    if (mode == 'P') != (b'PLTE' in kinds) or text > TEXT_BYTES:
        return None
    return h, w, ct, bits, mode, b''.join(p for k, p in chunks if k == b'IDAT')


def _rowbytes(w, mode, bits):
    return (w * CHANNELS[mode] * bits + 7) // 8


def accepts(info):
    """Whether the device accepts an eligible file: one zlib stream, nothing after it, exactly h * (rowbytes + 1)
    inflated bytes, and every filter type <= 4."""
    h, w, _, bits, mode, stream = info
    d = zlib.decompressobj()
    try:
        s = d.decompress(stream)
    except zlib.error:
        return False
    seg = _rowbytes(w, mode, bits) + 1
    return d.eof and not d.unused_data and len(s) == h * seg and max(s[::seg]) <= 4


def _unfilter(s, h, rowbytes, bpp):
    rows = np.frombuffer(s, np.uint8).reshape(h, rowbytes + 1)
    out = np.zeros((h, rowbytes), np.uint8)
    prev = np.zeros(rowbytes, np.int32)
    for y in range(h):
        f = rows[y, 0]
        r = rows[y, 1:].astype(np.int32)
        if f == 0:
            cur = r
        elif f == 2:
            cur = (r + prev) & 255
        elif f == 1:
            cur = np.empty_like(r)
            for k in range(min(bpp, rowbytes)):
                cur[k::bpp] = np.cumsum(r[k::bpp]) & 255
        else:
            cur = r.tolist()
            up = prev.tolist()
            for x in range(rowbytes):
                a = cur[x - bpp] if x >= bpp else 0
                b = up[x]
                if f == 3:
                    cur[x] = (cur[x] + ((a + b) >> 1)) & 255
                else:
                    c = up[x - bpp] if x >= bpp else 0
                    p = a + b - c
                    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                    cur[x] = (cur[x] + (a if pa <= pb and pa <= pc else b if pb <= pc else c)) & 255
            cur = np.array(cur, np.int32)
        out[y] = cur
        prev = cur
    return out


def decode(info):
    """Pillow's array of an accepted file: [h, w] (L, P) or [h, w, c] uint8; 2- and 4-bit grey scaled by 85 and 17."""
    h, w, _, bits, mode, stream = info
    c = CHANNELS[mode]
    rowbytes = _rowbytes(w, mode, bits)
    rows = _unfilter(zlib.decompress(stream), h, rowbytes, max(1, c * bits // 8))
    if bits == 8:
        return rows.reshape(h, w, c) if c > 1 else rows.reshape(h, w)
    px = np.unpackbits(rows, axis=1).reshape(h, -1, bits)[:, :w]
    vals = (px * (1 << np.arange(bits - 1, -1, -1))).sum(-1).astype(np.uint8)
    return vals * np.uint8(85 if bits == 2 else 17) if mode == 'L' else vals
