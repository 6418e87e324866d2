"""CPU restatement of the baseline JPEG that deva_b200_jpeg_encode writes (DESIGN §7, deva/utils/jpeg_encode.py): byte for
byte what Pillow's default ``Image.fromarray(rgb).save(f, 'JPEG', quality=q)`` writes through libjpeg(-turbo).

numpy only; all arithmetic is integer:
  * colour: libjpeg's ``jccolor.c`` fixed point, ``FIX(x) = int(x * 2^16 + 0.5)``;
  * edges: the last column is replicated to ``16 ceil(w / 16)``; the input is padded to an even row count (its last
    row repeated), luma is padded to ``16 ceil(h / 16)`` rows and the downsampled chroma planes to ``8 ceil(h / 16)``
    rows by repeating their own last row;
  * 4:2:0 downsampling ``(a + b + c + d + bias) >> 2``, bias 1, 2, 1, 2, ... along each output row;
  * level shift -128 and the ``islow`` integer DCT of ``jfdctint.c`` (output scaled by 8);
  * quantisation ``sign(c) ((|c| + 4 q) // (8 q))``.  libjpeg-turbo multiplies by a reciprocal instead; for every
    baseline divisor (8 q, q in [1, 255]) and every |c| < 2^15 that product equals this division;
  * MCU order Y00 Y01 Y10 Y11 Cb Cr; a luma block past ``ceil(w / 8)`` takes zero AC and the DC of the block to its
    left, a luma block row past ``ceil(h / 8)`` zero AC and the DC of the MCU's upper-right block;
  * Annex K Huffman tables, 1-bit fill, a 0x00 stuffed after every 0xFF byte of the scan;
  * SOI, APP0 (JFIF 1.01, no units, density 1x1), DQT 0, DQT 1, SOF0, DHT DC0 AC0 DC1 AC1, SOS, scan, EOI.
"""
import struct

import numpy as np

# Annex K.1: the luminance and chrominance quantisation tables, natural (row-major) order
STD_LUMA_Q = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99])
STD_CHROMA_Q = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
    47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32)

# Annex K.3: (code counts per length 1..16, symbols) of the DC / AC tables, luminance and chrominance
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
    0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0,
    0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28,
    0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
    0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
    0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5,
    0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
    0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa])
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
    0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0,
    0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26,
    0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87,
    0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5,
    0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
    0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa])


def _zigzag():
    """ZIGZAG[k] = natural index of the k-th coefficient in zigzag order."""
    order = sorted(((y, x) for y in range(8) for x in range(8)),
                   key=lambda p: (p[0] + p[1], p[1] if (p[0] + p[1]) % 2 == 0 else p[0]))
    return np.array([8 * y + x for y, x in order])


ZIGZAG = _zigzag()


def quant_tables(quality=75):
    """(luma, chroma) uint8 [64] in zigzag order: the Annex K tables scaled as ``jpeg_set_quality(q, baseline)``."""
    if not 1 <= quality <= 100:
        raise ValueError(f'quality must be in [1, 100], not {quality}')
    scale = 5000 // quality if quality < 50 else 200 - 2 * quality
    out = []
    for base in (STD_LUMA_Q, STD_CHROMA_Q):
        t = np.clip((base * scale + 50) // 100, 1, 255)
        out.append(t[ZIGZAG].astype(np.uint8))
    return tuple(out)


def huffman_codes(table):
    """(code, length) int64 [256] of every symbol of a (counts, symbols) table (canonical codes, Annex C)."""
    counts, symbols = table
    code_of, len_of = np.zeros(256, np.int64), np.zeros(256, np.int64)
    code, k = 0, 0
    for n, c in enumerate(counts, 1):
        for _ in range(c):
            code_of[symbols[k]], len_of[symbols[k]] = code, n
            code += 1
            k += 1
        code <<= 1
    return code_of, len_of


def ycc(img):
    """uint8 [h, w, 3] RGB -> int64 (Y, Cb, Cr) planes [h, w] (jccolor.c)."""
    fix = lambda x: int(x * 65536 + 0.5)  # noqa: E731
    r, g, b = (img[..., c].astype(np.int64) for c in range(3))
    half, off = 1 << 15, 128 << 16
    y = (fix(0.299) * r + fix(0.587) * g + fix(0.114) * b + half) >> 16
    cb = (-fix(0.16874) * r - fix(0.33126) * g + fix(0.5) * b + off + half - 1) >> 16
    cr = (fix(0.5) * r - fix(0.41869) * g - fix(0.08131) * b + off + half - 1) >> 16
    return y, cb, cr


def planes(img):
    """-> (Y [16 mh, 16 mw], Cb, Cr [8 mh, 8 mw]) int64, padded as libjpeg pads them."""
    h, w = img.shape[:2]
    mh, mw = -(-h // 16), -(-w // 16)
    cols = np.minimum(np.arange(16 * mw), w - 1)
    y, cb, cr = (p[:, cols] for p in ycc(img))
    luma = y[np.minimum(np.arange(16 * mh), h - 1)]
    even = np.minimum(np.arange(h + h % 2), h - 1)  # the input padded to an even row count
    bias = np.tile([1, 2], 4 * mw)
    chroma = []
    for p in (cb, cr):
        p = p[even]
        d = (p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2] + bias) >> 2
        chroma.append(d[np.minimum(np.arange(8 * mh), d.shape[0] - 1)])
    return luma, chroma[0], chroma[1]


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def fdct_islow(blocks):
    """int64 [n, 8, 8] level-shifted samples -> the jfdctint.c ``islow`` DCT [n, 8, 8] (natural order, scaled by 8)."""
    c_bits, p_bits = 13, 2
    d = blocks.astype(np.int64).copy()

    def one_pass(v, last):
        # v: [..., 8] along the transformed axis
        t0, t7 = v[..., 0] + v[..., 7], v[..., 0] - v[..., 7]
        t1, t6 = v[..., 1] + v[..., 6], v[..., 1] - v[..., 6]
        t2, t5 = v[..., 2] + v[..., 5], v[..., 2] - v[..., 5]
        t3, t4 = v[..., 3] + v[..., 4], v[..., 3] - v[..., 4]
        t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
        out = np.empty_like(v)
        if last:
            out[..., 0], out[..., 4] = _descale(t10 + t11, p_bits), _descale(t10 - t11, p_bits)
            sh = c_bits + p_bits
        else:
            out[..., 0], out[..., 4] = (t10 + t11) << p_bits, (t10 - t11) << p_bits
            sh = c_bits - p_bits
        z1 = (t12 + t13) * 4433
        out[..., 2] = _descale(z1 + t13 * 6270, sh)
        out[..., 6] = _descale(z1 - t12 * 15137, sh)
        z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
        z5 = (z3 + z4) * 9633
        t4, t5, t6, t7 = t4 * 2446, t5 * 16819, t6 * 25172, t7 * 12299
        z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
        out[..., 7] = _descale(t4 + z1 + z3, sh)
        out[..., 5] = _descale(t5 + z2 + z4, sh)
        out[..., 3] = _descale(t6 + z2 + z3, sh)
        out[..., 1] = _descale(t7 + z1 + z4, sh)
        return out

    d = one_pass(d, False)  # rows
    d = one_pass(d.transpose(0, 2, 1), True).transpose(0, 2, 1)  # columns
    return d


def _blocks(plane):
    """[8 a, 8 b] -> [a, b, 64] natural-order 8x8 blocks."""
    a, b = plane.shape[0] // 8, plane.shape[1] // 8
    return plane.reshape(a, 8, b, 8).transpose(0, 2, 1, 3).reshape(a, b, 64)


def _quantised(plane, table_zz):
    blk = _blocks(plane)
    a, b = blk.shape[:2]
    coef = fdct_islow(blk.reshape(-1, 8, 8) - 128).reshape(a, b, 64)[..., ZIGZAG]
    q = 8 * table_zz.astype(np.int64)
    return np.sign(coef) * ((np.abs(coef) + q // 2) // q)


def coefficients(img, quality=75):
    """int64 [n_mcu * 6, 64] quantised zigzag coefficients in scan order (Y00 Y01 Y10 Y11 Cb Cr per MCU, dummy blocks
    included) and the component (0 luma, 1 Cb, 2 Cr) of each block."""
    h, w = img.shape[:2]
    mh, mw = -(-h // 16), -(-w // 16)
    lq, cq = quant_tables(quality)
    luma, cb, cr = planes(img)
    y = _quantised(luma, lq)  # [2 mh, 2 mw, 64]
    if -(-w // 8) < 2 * mw:  # the last MCU column's right blocks are dummies
        y[:, -1, 1:] = 0
        y[:, -1, 0] = y[:, -2, 0]
    if -(-h // 8) < 2 * mh:  # the last MCU row's lower blocks are dummies: the DC of the MCU's upper-right block
        y[-1] = 0
        y[-1, :, 0] = y[-2, 1::2, 0].repeat(2)
    y = y.reshape(mh, 2, mw, 2, 64).transpose(0, 2, 1, 3, 4).reshape(mh, mw, 4, 64)
    c = np.stack([_quantised(cb, cq), _quantised(cr, cq)], 2)  # [mh, mw, 2, 64]
    coef = np.concatenate([y, c], 2).reshape(-1, 64)
    comp = np.tile([0, 0, 0, 0, 1, 2], mh * mw)
    return coef, comp


def _nbits(v):
    """Bits of |v| (0 for 0), elementwise."""
    a = np.abs(v)
    n = np.zeros(a.shape, np.int64)
    while (a > 0).any():
        n += a > 0
        a = a >> 1
    return n


def _tokens(coef, comp):
    """(value, length) int64 arrays of the scan's bit fields in order (code and magnitude bits joined)."""
    dc_tabs = [huffman_codes(DC_LUMA), huffman_codes(DC_CHROMA)]
    ac_tabs = [huffman_codes(AC_LUMA), huffman_codes(AC_CHROMA)]
    n = coef.shape[0]
    table = (comp > 0).astype(np.int64)

    # DC: differences against the previous block of the same component
    dc = coef[:, 0]
    prev = np.zeros(n, np.int64)
    for c in range(3):
        idx = np.nonzero(comp == c)[0]
        prev[idx[1:]] = dc[idx[:-1]]
    diff = dc - prev
    nb = _nbits(diff)
    mag = np.where(diff < 0, diff - 1, diff) & ((1 << nb) - 1)
    dcode = np.where(table == 0, dc_tabs[0][0][nb], dc_tabs[1][0][nb])
    dlen = np.where(table == 0, dc_tabs[0][1][nb], dc_tabs[1][1][nb])
    keys = [np.arange(n) * 8192]
    vals, lens = [(dcode << nb) | mag], [dlen + nb]

    # AC: every nonzero coefficient with the zero runs (ZRL per 16) before it, then EOB unless k = 63 is nonzero
    ac = coef[:, 1:]
    b, k = np.nonzero(ac)
    k = k + 1
    v = ac[b, k - 1]
    first = np.ones(len(b), bool)
    first[1:] = b[1:] != b[:-1]
    prev_k = np.where(first, 0, np.concatenate([[0], k[:-1]]))
    run = k - prev_k - 1
    nb = _nbits(v)
    mag = np.where(v < 0, v - 1, v) & ((1 << nb) - 1)
    sym = ((run & 15) << 4) | nb
    t = table[b]
    acode = np.where(t == 0, ac_tabs[0][0][sym], ac_tabs[1][0][sym])
    alen = np.where(t == 0, ac_tabs[0][1][sym], ac_tabs[1][1][sym])
    keys.append(b * 8192 + k * 64 + 8)
    vals.append((acode << nb) | mag)
    lens.append(alen + nb)
    zrl = run >> 4
    zi = np.repeat(np.arange(len(b)), zrl)
    sub = np.arange(len(zi)) - np.repeat(np.cumsum(zrl) - zrl, zrl)
    zt = t[zi]
    keys.append(b[zi] * 8192 + k[zi] * 64 + sub)
    vals.append(np.where(zt == 0, ac_tabs[0][0][0xf0], ac_tabs[1][0][0xf0]))
    lens.append(np.where(zt == 0, ac_tabs[0][1][0xf0], ac_tabs[1][1][0xf0]))
    eob = np.nonzero(coef[:, 63] == 0)[0]
    keys.append(eob * 8192 + 64 * 64)
    vals.append(np.where(table[eob] == 0, ac_tabs[0][0][0], ac_tabs[1][0][0]))
    lens.append(np.where(table[eob] == 0, ac_tabs[0][1][0], ac_tabs[1][1][0]))

    order = np.argsort(np.concatenate(keys), kind='stable')
    return np.concatenate(vals)[order], np.concatenate(lens)[order]


def scan(coef, comp):
    """The entropy-coded segment: the tokens' bits MSB first, 1-bit fill, 0x00 stuffed after every 0xFF."""
    vals, lens = _tokens(coef, comp)
    total = int(lens.sum())
    start = np.cumsum(lens) - lens
    tok = np.repeat(np.arange(len(lens)), lens)
    j = np.arange(total) - start[tok]
    bits = ((vals[tok] >> (lens[tok] - 1 - j)) & 1).astype(np.uint8)
    bits = np.concatenate([bits, np.ones(-total % 8, np.uint8)])
    data = np.packbits(bits)
    ff = np.nonzero(data == 0xff)[0]
    return np.insert(data, ff + 1, 0).tobytes()


def _segment(marker, body):
    return struct.pack('>BBH', 0xff, marker, len(body) + 2) + body


def headers(h, w, quality=75):
    """Every marker segment before the scan: SOI .. SOS."""
    lq, cq = quant_tables(quality)
    out = b'\xff\xd8' + _segment(0xe0, b'JFIF\0' + bytes([1, 1, 0]) + struct.pack('>HHBB', 1, 1, 0, 0))
    out += _segment(0xdb, b'\0' + lq.tobytes()) + _segment(0xdb, b'\1' + cq.tobytes())
    out += _segment(0xc0, struct.pack('>BHHB', 8, h, w, 3) + bytes([1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for tc_th, (counts, symbols) in ((0x00, DC_LUMA), (0x10, AC_LUMA), (0x01, DC_CHROMA), (0x11, AC_CHROMA)):
        out += _segment(0xc4, bytes([tc_th] + counts + symbols))
    out += _segment(0xda, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))
    return out


def encode_jpeg(img, quality=75):
    """The JPEG file of uint8 RGB ``img`` [h, w, 3] at ``quality``."""
    img = np.asarray(img)
    assert img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3, (img.dtype, img.shape)
    h, w = img.shape[:2]
    coef, comp = coefficients(img, quality)
    return headers(h, w, quality) + scan(coef, comp) + b'\xff\xd9'
