"""Restatement of the device JPEG decoder (deva/utils/jpeg_decode.py, csrc/jpeg_decode.cu) in numpy: the sequential
decode of a device-eligible file and the status the device gives it.  The file's structure is read by the package's
``parse`` (the eligibility rule); the Huffman decode (bit by bit, canonical codes), the DC prediction, jidctint.c's
islow IDCT, libjpeg-turbo's fancy upsampling and jdcolor.c's YCbCr -> RGB are written out again here, so that
tests/test_jpeg_decode_cpu.py can pin them to Pillow."""
import numpy as np

from deva.utils.jpeg_decode import HUFF_WORDS, NATURAL, parse

OK, BAD_CODE, BAD_CATEGORY, RUN_PAST_63, SHORT_STREAM, TRAILING, RANGE = 0, 2, 3, 4, 5, 6, 7
COEF_LIMIT = 16383


def _tables(hd, c, ac):
    t = hd.tables[(2 * c + ac) * HUFF_WORDS:(2 * c + ac + 1) * HUFF_WORDS]
    return t[512:530], t[530:548], t[548:]


def _coefficients(hd):
    """-> (status, int16 [blocks, 64] natural-order coefficients in MCU order)."""
    bpm = hd.hy * hd.vy + 2
    comp = [0] * (hd.hy * hd.vy) + [1, 2]
    coef = np.zeros((hd.blocks, 64), np.int16)
    tabs = [[_tables(hd, c, ac) for ac in (0, 1)] for c in range(3)]
    for a, b, m0, m in hd.intervals:
        bits = np.unpackbits(hd.scan[a:b])
        n, pos, pred = len(bits), 0, [0, 0, 0]

        def take(k):
            nonlocal pos
            if pos + k > n:
                raise EOFError
            v = 0
            for i in range(k):
                v = v << 1 | int(bits[pos + i])
            pos += k
            return v

        def symbol(t):
            maxcode, valoff, vals = t
            code = 0
            for length in range(1, 17):
                code = code << 1 | take(1)
                if code <= maxcode[length]:
                    return int(vals[code + valoff[length]])
            return None

        def extend(v, s):
            return v - (1 << s) + 1 if s and v < 1 << (s - 1) else v
        try:
            for blk in range(m0 * bpm, (m0 + m) * bpm):
                c = comp[blk % bpm]
                s = symbol(tabs[c][0])
                if s is None:
                    return BAD_CODE, None
                if s > 11:
                    return BAD_CATEGORY, None
                pred[c] += extend(take(s), s)
                coef[blk, 0] = np.int32(pred[c]).astype(np.int16)
                k = 1
                while k < 64:
                    rs = symbol(tabs[c][1])
                    if rs is None:
                        return BAD_CODE, None
                    r, s = rs >> 4, rs & 15
                    if s:
                        if s > 10:
                            return BAD_CATEGORY, None
                        k += r
                        if k > 63:
                            return RUN_PAST_63, None
                        coef[blk, NATURAL[k]] = extend(take(s), s)
                        k += 1
                    elif r == 15:
                        k += 16
                        if k > 64:
                            return RUN_PAST_63, None
                    else:
                        break
        except EOFError:
            return SHORT_STREAM, None
        if n - pos >= 8:
            return TRAILING, None
    return OK, coef


def idct_islow(coef, quant):
    """int16 [n, 64] coefficients, int [64] natural-order quantisation -> (uint8 [n, 8, 8] samples, bool [n]: the
    block leaves the range where libjpeg-turbo's C and SIMD islow paths agree)."""
    x = coef.astype(np.int64).reshape(-1, 8, 8) * np.asarray(quant, np.int64).reshape(8, 8)
    bad = np.abs(x).reshape(len(x), -1).max(1, initial=0) > COEF_LIMIT

    def one_d(v, rnd, shift, dc_bias=0):
        # v[..., k, :]: input k of the 1-D transform along axis -2
        z2, z3 = v[..., 2, :], v[..., 6, :]
        z1 = (z2 + z3) * 4433
        tmp2, tmp3 = z1 - z3 * 15137, z1 + z2 * 6270
        z2, z3 = v[..., 0, :] + dc_bias, v[..., 4, :]
        tmp0, tmp1 = (z2 + z3) << 13, (z2 - z3) << 13
        tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
        t0, t1, t2, t3 = v[..., 7, :], v[..., 5, :], v[..., 3, :], v[..., 1, :]
        z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
        z5 = (z3 + z4) * 9633
        t0, t1, t2, t3 = t0 * 2446, t1 * 16819, t2 * 25172, t3 * 12299
        z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
        t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
        out = [tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0, tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3]
        return np.stack([(o + rnd) >> shift for o in out], -2)
    ws = one_d(x, 1 << 10, 11)                                      # columns: [n, row, col]
    bad |= np.abs(ws).reshape(len(ws), -1).max(1, initial=0) > COEF_LIMIT
    out = one_d(np.swapaxes(ws, 1, 2), 0, 18, dc_bias=1 << 4)       # rows
    out = np.swapaxes(out, 1, 2)
    bad |= ((out > 511) | (out < -512)).reshape(len(out), -1).any(1)
    return (np.clip(out, -128, 127) + 128).astype(np.uint8), bad


def _planes(hd, coef):
    bpm = hd.hy * hd.vy + 2
    mx = (hd.w + 8 * hd.hy - 1) // (8 * hd.hy)
    my = (hd.h + 8 * hd.vy - 1) // (8 * hd.vy)
    quant = hd.tables[6 * HUFF_WORDS:].reshape(3, 64)
    blocks = coef.reshape(my, mx, bpm, 64)
    planes, bad = [], False
    ny = hd.hy * hd.vy
    y = blocks[:, :, :ny].reshape(my, mx, hd.vy, hd.hy, 64)
    samples, b = idct_islow(y.reshape(-1, 64), quant[0])
    bad |= b.any()
    planes.append(samples.reshape(my, mx, hd.vy, hd.hy, 8, 8).transpose(0, 2, 4, 1, 3, 5).reshape(my * hd.vy * 8,
                                                                                                    mx * hd.hy * 8))
    for c in (1, 2):
        samples, b = idct_islow(blocks[:, :, ny + c - 1].reshape(-1, 64), quant[c])
        bad |= b.any()
        planes.append(samples.reshape(my, mx, 8, 8).transpose(0, 2, 1, 3).reshape(my * 8, mx * 8))
    return planes, bad


def _upsample(hd, p):
    """A chroma plane at full size (libjpeg-turbo's h2v1 / h2v2 fancy upsampling, replication when the chroma width is at
    most 2)."""
    h, w = hd.h, hd.w
    if hd.hy == 1:
        return p[:h, :w].astype(np.int64)
    dw, dh = (w + 1) // 2, (h + 1) // 2 if hd.vy == 2 else h
    x = np.arange(w)
    i = x >> 1
    yy = np.arange(h)
    if dw <= 2:
        return p[(yy >> 1) if hd.vy == 2 else yy][:, i].astype(np.int64)
    ni = np.where(x & 1, np.minimum(i + 1, dw - 1), np.maximum(i - 1, 0))
    p = p.astype(np.int64)
    if hd.vy == 1:
        return (3 * p[:h, i] + p[:h, ni] + np.where(x & 1, 2, 1)) >> 2
    j = yy >> 1
    nj = np.where(yy & 1, np.minimum(j + 1, dh - 1), np.maximum(j - 1, 0))
    c0 = 3 * p[j][:, i] + p[nj][:, i]
    c1 = 3 * p[j][:, ni] + p[nj][:, ni]
    return (3 * c0 + c1 + np.where(x & 1, 7, 8)) >> 4


def ycc_to_rgb(y, cb, cr):
    xcb, xcr = cb - 128, cr - 128
    r = y + ((91881 * xcr + 32768) >> 16)
    g = y + ((-46802 * xcr - 22554 * xcb + 32768) >> 16)
    b = y + ((116130 * xcb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(data):
    """-> (status, uint8 [h, w, 3] or None) for a device-eligible file; None for any other file."""
    hd = parse(data)
    if hd is None:
        return None
    st, coef = _coefficients(hd)
    if st:
        return st, None
    planes, bad = _planes(hd, coef)
    if bad:
        return RANGE, None
    y = planes[0][:hd.h, :hd.w].astype(np.int64)
    return OK, ycc_to_rgb(y, _upsample(hd, planes[1]), _upsample(hd, planes[2]))
