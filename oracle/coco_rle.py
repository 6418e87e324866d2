"""CPU restatement of COCO's compressed RLE, the strings ``pycocotools.mask.encode(np.asfortranarray(m))`` stores and
deva_b200_rle_encode writes (DESIGN §7, deva/utils/rle_encode.py).

Pure Python and numpy, following pycocotools' maskApi.c:
  * ``rleEncode``: scan the mask in column-major order (position ``p = x * h + y``) starting from ``prev = 0``; every
    change of value closes the current run, and the last run is closed at the end.  The first count is the leading
    run of zeros (0 when pixel 0 is set); an all-zero mask is ``[h * w]``;
  * ``rleToString``: count ``i`` is written as ``x = cnts[i] - cnts[i - 2]`` when ``i > 2`` (not ``i >= 2``) and as
    ``cnts[i]`` otherwise, in 5-bit chunks, low bits first, each as ``chr(48 + c)`` with 0x20 set on every chunk but
    the last.  After ``x >>= 5`` (arithmetic) the chunks go on while ``x != -1`` if the chunk's 0x10 bit is set, else
    while ``x != 0``: the values are sign-terminated;
  * the result is ``{'size': [h, w], 'counts': str}``.
``decode`` restates ``rleFrString`` and ``rleDecode`` for round trips.
"""
import numpy as np


def counts(mask: np.ndarray) -> list:
    """The run lengths of a 2-D mask (nonzero = set) in column-major order, starting with a run of zeros."""
    m = np.asarray(mask)
    assert m.ndim == 2, m.shape
    flat = (m != 0).reshape(-1, order='F').astype(np.int8)
    n = flat.size
    change = np.flatnonzero(np.diff(flat, prepend=0))  # positions where the value differs from the one before
    edges = np.concatenate([[0], change, [n]])
    return [int(c) for c in np.diff(edges)]


def _chars(x: int) -> str:
    out = []
    more = True
    while more:
        c = x & 0x1f
        x >>= 5
        more = (x != -1) if c & 0x10 else (x != 0)
        if more:
            c |= 0x20
        out.append(chr(48 + c))
    return ''.join(out)


def counts_to_string(cnts) -> str:
    """rleToString: the compressed string of a list of run lengths."""
    return ''.join(_chars(int(cnts[i]) - (int(cnts[i - 2]) if i > 2 else 0)) for i in range(len(cnts)))


def string_to_counts(s: str) -> list:
    """rleFrString: the run lengths of a compressed string."""
    cnts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = ord(s[p]) - 48
            x |= (c & 0x1f) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(cnts) > 2:
            x += cnts[-2]
        cnts.append(x)
    return cnts


def encode(mask: np.ndarray) -> dict:
    """``pycocotools.mask.encode(np.asfortranarray(mask))`` with its counts decoded to str."""
    h, w = np.asarray(mask).shape
    return {'size': [int(h), int(w)], 'counts': counts_to_string(counts(mask))}


def decode(rle: dict) -> np.ndarray:
    """rleDecode: the uint8 [h, w] mask of ``{'size': [h, w], 'counts': str}``."""
    h, w = rle['size']
    cnts = string_to_counts(rle['counts'])
    assert sum(cnts) == h * w, (sum(cnts), h, w)
    flat = np.repeat(np.arange(len(cnts)) % 2, cnts).astype(np.uint8)
    return flat.reshape((h, w), order='F')


def encode_ids(ids: np.ndarray, seg_ids) -> list:
    """One ``encode(ids == i)`` per entry of ``seg_ids``: what deva_b200_rle_encode writes for an id map."""
    ids = np.asarray(ids)
    return [encode(ids == int(i)) for i in seg_ids]
