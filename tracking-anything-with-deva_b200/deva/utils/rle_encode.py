"""COCO RLE of an id map's segments encoded on the device (``deva_b200_rle_encode``): an opt-in replacement for the
per-segment ``pycocotools.mask.encode`` loop of the BURST result saver, selected by ``rle_encoder='device'`` or
``DEVA_B200_RLE_ENCODER=device``.

``encode_rle(ids, seg_ids)`` equals ``[pycocotools.mask.encode(np.asfortranarray(ids == i)) for i in seg_ids]`` with
each ``counts`` decoded to str, string for string (oracle/coco_rle.py restates the format):
  * the runs of the mask in column-major order, starting with a run of zeros (0 when pixel 0 is set);
  * count ``i`` written as ``cnts[i] - cnts[i - 2]`` when ``i > 2``, else ``cnts[i]``, in 5-bit chunks, low bits first,
    each ``chr(48 + c)`` with 0x20 on every chunk but the last, ended when the rest is the chunk's sign extension.
All segments come from one pass over the map; a repeated id gets the same string again, and an id absent from the map
the string of ``[h * w]``.

``encode_rle_async`` uploads the seg ids and enqueues the encode and one copy of the offsets and the strings' first
``PREFIX`` bytes on the current stream without synchronising; the returned ``Pending``'s ``result()`` waits for them
(and fetches the rest of longer strings; deva/utils/device_download.py).  Importing this module neither imports
pycocotools nor initialises CUDA.
"""
import functools
from typing import List, Optional

import numpy as np
import torch

from deva._native import MAX_SEGMENT_CHANNELS
from deva.utils import device_download

ENCODERS = ('pycocotools', 'device')
ENV = 'DEVA_B200_RLE_ENCODER'
PREFIX = 1024 * 1024  # string bytes copied with the encode; result() fetches the rest
MAX_PIXELS = 2**31 - 1  # pycocotools' counts are 32-bit
_INT_DTYPES = (torch.bool, torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64)


def resolve_encoder(rle_encoder: Optional[str] = None) -> str:
    """``rle_encoder``, or the environment's ``DEVA_B200_RLE_ENCODER`` when it is None ('pycocotools' when unset)."""
    return device_download.resolve(rle_encoder, 'rle_encoder', ENV, ENCODERS, 'pycocotools')


def host_bytes(n: int) -> int:
    """Bytes of the pinned buffer ``encode_rle_async`` needs for ``n`` seg ids: the ids, the offsets, the prefix."""
    return 16 * n + 8 + PREFIX


def _strings(h: int, w: int, offsets: List[int], data: bytes) -> List[dict]:
    text = data.decode('ascii')
    return [{'size': [h, w], 'counts': text[offsets[j]:offsets[j + 1]]} for j in range(len(offsets) - 1)]


def _as_device_ids(ids) -> torch.Tensor:
    if isinstance(ids, np.ndarray):
        if not (ids.ndim == 2 and (ids.dtype == np.bool_ or np.issubdtype(ids.dtype, np.signedinteger) or
                                   ids.dtype in (np.uint8, np.uint16, np.uint32))):
            raise ValueError(f'an id map is an integer array [h, w], not {ids.dtype} {ids.shape}')
        _check_shape(ids.shape)
        return device_download.upload(ids, np.int64)
    if not (isinstance(ids, torch.Tensor) and ids.is_cuda and ids.dtype in _INT_DTYPES and ids.dim() == 2):
        desc = f'{ids.dtype} {tuple(ids.shape)} on {ids.device}' if isinstance(ids, torch.Tensor) else type(ids)
        raise ValueError(f'an id map is a CUDA integer tensor [h, w] or a numpy array, not {desc}')
    _check_shape(ids.shape)
    return ids.to(torch.int64).contiguous()


def _check_shape(shape):
    h, w = int(shape[0]), int(shape[1])
    if not (h >= 1 and w >= 1 and h * w <= MAX_PIXELS):
        raise ValueError(f'an id map has 1 <= h, w and h * w < 2^31, not {h} x {w}')


def _as_id_list(seg_ids) -> List[int]:
    if isinstance(seg_ids, torch.Tensor):
        if seg_ids.is_cuda:
            raise ValueError('seg_ids are host values (a sequence, numpy array or CPU tensor), not a CUDA tensor')
        seg_ids = seg_ids.tolist()
    out = []
    for i in np.asarray(seg_ids, dtype=object).reshape(-1).tolist():
        if isinstance(i, (bool, np.bool_)) or not isinstance(i, (int, np.integer)):
            raise ValueError(f'seg ids are integers, not {i!r}')
        if not -2**63 <= int(i) < 2**63:
            raise ValueError(f'seg id {i} does not fit in int64')
        out.append(int(i))
    if len(out) > MAX_SEGMENT_CHANNELS:
        raise ValueError(f'at most {MAX_SEGMENT_CHANNELS} seg ids per encode, not {len(out)}')
    return out


def encode_rle_async(ids, seg_ids, host: Optional[torch.Tensor] = None) -> device_download.Pending:
    """Enqueues the RLE of ``ids == i`` for every ``i`` in ``seg_ids`` on the current stream; never synchronises the
    host.  ids: integer [h, w] (a CUDA tensor, or a numpy array that is uploaded); seg_ids: host integers.  host:
    optional pinned uint8 buffer of at least ``host_bytes(len(seg_ids))`` bytes through which the seg ids go up and the
    offsets and the strings' first bytes come back (one is allocated otherwise); it must stay untouched until
    ``result()`` returns, which gives one ``{'size': [h, w], 'counts': str}`` per seg id."""
    seg = _as_id_list(seg_ids)
    ids = _as_device_ids(ids)
    h, w = int(ids.shape[0]), int(ids.shape[1])
    n = len(seg)
    if n == 0:
        return device_download.Pending(lambda *_: [])
    from deva import _native
    bound = _native.rle_bound(h, w, n)
    at = 16 * n + 8  # [seg ids | offsets | strings | workspace], the first three as in the host buffer
    dev, out, ws = device_download.buffer(at, bound, _native.rle_workspace_bytes(h, w, n), ids.device)
    host = device_download.pinned(host, at + min(PREFIX, bound))
    host[:8 * n].view(torch.int64).numpy()[:] = seg
    dev[:8 * n].copy_(host[:8 * n], non_blocking=True)
    _native.rle_encode(ids, dev[:8 * n].view(torch.int64), ws, out, dev[8 * n:at].view(torch.int64))
    return device_download.enqueue(functools.partial(_strings, h, w), dev, (8 * n, at), bound, PREFIX, host)


def encode_rle(ids, seg_ids) -> List[dict]:
    """One ``{'size': [h, w], 'counts': str}`` per entry of ``seg_ids`` (see ``encode_rle_async``); waits for the
    device."""
    return encode_rle_async(ids, seg_ids).result()
