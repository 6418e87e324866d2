"""CPU restatement of the PNG format that deva_b200_png_encode writes (DESIGN §7, deva/utils/png_encode.py).

numpy and the standard library only; byte for byte what the device writes:
  * the zlib stream of the image's filtered bytes ``s`` (every row ``[2] + Up-filtered row``, row 0 against zeros);
  * each row segment of ``s`` is tokenised greedily on its own: at position i the candidate distances are {1, bpp}, a
    match's length is the run of ``s[j] == s[j - d]`` (``j - d >= 0`` in stream coordinates, ``j`` within the row
    segment), capped at 258; the longer candidate wins, a tie goes to the smaller distance; a length >= 3 is a match,
    anything else the literal ``s[i]``;
  * one fixed-Huffman block (BFINAL = 1, BTYPE = 01), end-of-block, zero padding, header 0x78 0x01, Adler-32 trailer;
  * chunks: signature, IHDR, PLTE (P only), one IDAT, IEND; bit depth and PLTE follow Pillow's writer for the image.
"""
import struct
import zlib

import numpy as np

SIGNATURE = b'\x89PNG\r\n\x1a\n'
MAX_MATCH = 258
LBASE = np.array([3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163,
                  195, 227, 258])
LEXT = np.array([0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0])


def layout(mode, palette=None):
    """(colour type, bit depth, PLTE bytes or None) Pillow's PNG writer picks for an image of ``mode`` whose palette was
    set by ``putpalette(palette)``: a P palette of <= 2 / 4 / 16 colours is written at 1 / 2 / 4 bits."""
    if mode == 'L':
        return 0, 8, None
    if mode == 'RGB':
        return 2, 8, None
    assert mode == 'P', mode
    from PIL import Image
    im = Image.new('P', (1, 1))
    if palette is not None:
        im.putpalette(palette)
    colors = max(min(len(im.palette.getdata()[1]) // 3, 256), 1) if im.palette else 256
    bits = 1 if colors <= 2 else 2 if colors <= 4 else 4 if colors <= 16 else 8
    plte = im.im.getpalette('RGB')[:colors * 3]
    return 3, bits, plte + b'\0' * (colors * 3 - len(plte))


def raw_rows(img, bits):
    """uint8 [h, row bytes]: the image's rows as Pillow packs them.  Sub-byte rows are packed MSB-first with zero padding;
    at 2 and 4 bits a pixel keeps ``v & (2^bits - 1)``, at 1 bit it is ``v != 0`` (Pillow's bilevel packer)."""
    h, w = img.shape[:2]
    a = img.reshape(h, -1).astype(np.uint8)
    if bits == 8:
        return a
    ppb = 8 // bits
    pad = (-w) % ppb
    a = (a != 0).astype(np.uint8) if bits == 1 else a & ((1 << bits) - 1)
    v = np.pad(a, ((0, 0), (0, pad))).reshape(h, -1, ppb).astype(np.uint16)
    shifts = (8 - bits * (np.arange(ppb) + 1)).astype(np.uint16)
    return (v << shifts).sum(-1).astype(np.uint8)


def filtered(img, bits):
    """s as uint8 [h, row bytes + 1]: filter byte 2 (Up) and the Up-filtered row."""
    raw = raw_rows(img, bits)
    prev = np.vstack([np.zeros((1, raw.shape[1]), np.uint8), raw[:-1]])
    return np.hstack([np.full((raw.shape[0], 1), 2, np.uint8), raw - prev])


def _runs(s, d):
    """int32 [h, seg]: run of s[j] == s[j - d] from each position to the end of its row segment (not capped)."""
    h, seg = s.shape
    flat = s.reshape(-1)
    eq = np.zeros(flat.size, bool)
    eq[d:] = flat[d:] == flat[:-d]
    eq = eq.reshape(h, seg)
    # run[i] = (index of the first False at or after i) - i, with a False sentinel at the segment's end
    pos = np.where(~eq, np.arange(seg)[None, :], seg)
    first_false = np.minimum.accumulate(pos[:, ::-1], axis=1)[:, ::-1]
    return (first_false - np.arange(seg)[None, :]).astype(np.int32)


def tokens(s, bpp):
    """Greedy tokens of every row -> (length int32 [n], distance int32 [n], literal uint8 [n]) in stream order; a
    length of 1 marks a literal."""
    h, seg = s.shape
    best = np.minimum(_runs(s, 1), MAX_MATCH)
    dist = np.ones_like(best)
    if bpp > 1:
        other = np.minimum(_runs(s, bpp), MAX_MATCH)
        take = other > best
        best = np.where(take, other, best)
        dist = np.where(take, bpp, dist)
    step = np.where(best >= 3, best, 1).reshape(-1)
    dist, best = dist.reshape(-1), best.reshape(-1)
    # the walk: from each row start, i -> i + step[i]; literal stretches are taken whole
    is_match = step > 1
    next_match = np.where(is_match, np.arange(step.size), step.size)
    next_match = np.minimum.accumulate(next_match[::-1])[::-1]
    starts = []
    for y in range(h):
        i, end = y * seg, (y + 1) * seg
        while i < end:
            m = min(int(next_match[i]), end)
            if m > i:
                starts.append(np.arange(i, m))
                i = m
                continue
            starts.append(np.array([i]))
            i += int(step[i])
    starts = np.concatenate(starts)
    lengths = np.where(is_match[starts], best[starts], 1).astype(np.int32)
    return lengths, dist[starts].astype(np.int32), s.reshape(-1)[starts]


def _reverse(code, n):
    code, n = np.asarray(code, np.int64), np.asarray(n, np.int64)
    out = np.zeros_like(code)
    for k in range(9):
        out |= ((code >> k) & 1) << np.maximum(n - 1 - k, 0)  # bits k >= n of a code are 0
    return np.where(n > 0, out, 0)


def deflate_fields(lengths, dists, literals):
    """(value, bit count) of every field of the block, LSB-first, in stream order (header and end-of-block included)."""
    lit = literals.astype(np.int64)
    lit_code = np.where(lit <= 143, 0x30 + lit, 0x190 + lit - 144)
    lit_n = np.where(lit <= 143, 8, 9)
    k = np.where(lengths == 258, 28, np.searchsorted(LBASE[:28], lengths, side='right') - 1)
    sym = 257 + k
    len_code = np.where(sym <= 279, sym - 256, 0xC0 + sym - 280)
    len_n = np.where(sym <= 279, 7, 8)
    match = lengths >= 3
    n = lengths.size
    # three fields per token: (symbol, extra bits, distance); unused fields have 0 bits
    val = np.zeros((n, 3), np.int64)
    nb = np.zeros((n, 3), np.int64)
    val[:, 0] = np.where(match, _reverse(len_code, len_n), _reverse(lit_code, lit_n))
    nb[:, 0] = np.where(match, len_n, lit_n)
    val[:, 1] = np.where(match, lengths - LBASE[np.clip(k, 0, 28)], 0)
    nb[:, 1] = np.where(match, LEXT[np.clip(k, 0, 28)], 0)
    val[:, 2] = np.where(match, _reverse(dists - 1, 5), 0)
    nb[:, 2] = np.where(match, 5, 0)
    val = np.concatenate([[3], val.reshape(-1), [0]])  # BFINAL = 1, BTYPE = 01; end-of-block is seven 0 bits
    nb = np.concatenate([[3], nb.reshape(-1), [7]])
    return val, nb


def pack_bits(val, nb):
    """Bytes of the LSB-first concatenation of the fields, zero-padded to a byte."""
    keep = nb > 0
    val, nb = val[keep], nb[keep]
    total = int(nb.sum())
    starts = np.cumsum(nb) - nb
    owner = np.repeat(np.arange(nb.size), nb)
    bit = (val[owner] >> (np.arange(total) - starts[owner])) & 1
    return np.packbits(bit.astype(np.uint8), bitorder='little').tobytes()


def zlib_stream(img, bits, bpp):
    s = filtered(img, bits)
    body = pack_bits(*deflate_fields(*tokens(s, bpp)))
    return b'\x78\x01' + body + struct.pack('>I', zlib.adler32(s.tobytes()))


def bound(h, row_bytes):
    """Hard bound on the zlib stream's size: every byte of s a 9-bit literal."""
    n = h * (row_bytes + 1)
    return (3 + 9 * n + 7 + 7) // 8 + 6


def _chunk(kind, data):
    return struct.pack('>I', len(data)) + kind + data + struct.pack('>I', zlib.crc32(kind + data))


def encode_png(img, mode, palette=None):
    """PNG file bytes of uint8 [h, w] (L, P) or [h, w, 3] (RGB) ``img``."""
    img = np.ascontiguousarray(img, np.uint8)
    assert img.ndim == (3 if mode == 'RGB' else 2) and (mode != 'RGB' or img.shape[2] == 3), (mode, img.shape)
    h, w = img.shape[:2]
    colour, bits, plte = layout(mode, palette)
    bpp = 3 if mode == 'RGB' else 1
    out = SIGNATURE + _chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, bits, colour, 0, 0, 0))
    if plte is not None:
        out += _chunk(b'PLTE', plte)
    return out + _chunk(b'IDAT', zlib_stream(img, bits, bpp)) + _chunk(b'IEND', b'')
