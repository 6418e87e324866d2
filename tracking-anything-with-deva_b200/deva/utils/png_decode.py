"""PNG files decoded on the device (``deva_b200_png_decode``): an opt-in replacement for Pillow's PNG reader in the
post-processing passes, selected by ``png_decoder='device'`` or ``DEVA_B200_PNG_DECODER=device``.

For every file the result is exactly what Pillow gives: ``np.asarray(Image.open(f))`` as a CUDA tensor, or the
exception Pillow raises.  The device takes the plain, well-formed case and every other file is read by Pillow, so none
of Pillow's quirks (zero-filled rows of a short stream, ignored trailing data, an unchecked IDAT CRC, ...) is restated
here.  A file is device-eligible (``parse``, decided on the host) when:
  * it has the PNG signature; every chunk is in bounds with a valid CRC; IHDR comes first and IEND last with nothing
    after it; the IDAT chunks are consecutive and there is at least one;
  * IHDR has w, h >= 1, compression 0, filter method 0 and interlace 0, and ``w * h <= Image.MAX_IMAGE_PIXELS`` (so the
    decompression-bomb warning and error stay Pillow's);
  * (colour type, bit depth) is grey at 2, 4 or 8 bits (Pillow's mode L, scaling 2-bit by 85 and 4-bit by 17), palette
    at 1, 2, 4 or 8 (mode P, unscaled indices) with one PLTE of 1 to 256 entries before the IDATs, RGB 8 or RGBA 8.
    1-bit grey (mode 1, a bool array), LA, 16-bit, Adam7 and APNG are Pillow's;
  * every other chunk is one of ``ANCILLARY``, at most once (tEXt any number of times, up to ``TEXT_BYTES`` in all),
    with the length the PNG specification gives it, before the IDATs (tEXt and tIME may also follow them).
tests/test_png_decode_cpu.py checks that each of these chunks leaves Pillow's array unchanged.  The device then accepts
a file (status 0) only when its stream is one well-formed zlib stream of exactly ``h * (rowbytes + 1)`` bytes with a
matching Adler-32 and nothing after it, and every row's filter type is at most 4 (csrc/inflate.cuh); any nonzero
status sends the file to Pillow.

Files go to the device in batches of at most ``BUDGET`` decoded bytes: one pinned staging copy of the batch's
descriptors and streams, one launch (``enqueue``), and one host synchronisation to read the statuses.  Importing this module does
not initialise CUDA.
"""
import struct
import zlib
from typing import List, NamedTuple, Optional

import numpy as np
import torch

from deva.utils import device_decode, device_download

DECODERS = ('pil', 'device')
ENV = 'DEVA_B200_PNG_DECODER'
SIGNATURE = b'\x89PNG\r\n\x1a\n'
BUDGET = 256 << 20  # decoded bytes (arrays and filtered streams) of one batch
TEXT_BYTES = 1 << 20  # tEXt bytes of an eligible file
ANCILLARY = (b'tRNS', b'gAMA', b'cHRM', b'sRGB', b'pHYs', b'sBIT', b'bKGD', b'tEXt', b'tIME')
_AFTER_IDAT = (b'tEXt', b'tIME')
_MODES = {(0, 2): 'L', (0, 4): 'L', (0, 8): 'L', (3, 1): 'P', (3, 2): 'P', (3, 4): 'P', (3, 8): 'P', (2, 8): 'RGB',
          (6, 8): 'RGBA'}
_CHANNELS = {'L': 1, 'P': 1, 'RGB': 3, 'RGBA': 4}
_ALIGN = 16


class Header(NamedTuple):
    """A device-eligible file: its shape, format and the byte ranges of its IDAT data."""
    h: int
    w: int
    colour_type: int
    bits: int
    mode: str
    idat: tuple

    @property
    def shape(self):
        c = _CHANNELS[self.mode]
        return (self.h, self.w) if c == 1 else (self.h, self.w, c)

    @property
    def nbytes(self):
        return self.h * self.w * _CHANNELS[self.mode]

    def stream(self, data) -> bytes:
        return b''.join(data[a:b] for a, b in self.idat)


def resolve_decoder(png_decoder: Optional[str] = None) -> str:
    """``png_decoder``, or the environment's ``DEVA_B200_PNG_DECODER`` when it is None ('pil' when that is unset)."""
    return device_download.resolve(png_decoder, 'png_decoder', ENV, DECODERS, 'pil')


def _ancillary_ok(kind, n, mode, palette_entries):
    if kind in (b'gAMA', b'cHRM', b'sRGB', b'pHYs', b'tIME'):
        return n == {b'gAMA': 4, b'cHRM': 32, b'sRGB': 1, b'pHYs': 9, b'tIME': 7}[kind]
    if kind == b'tRNS':
        return (mode == 'P' and 1 <= n <= palette_entries) or n == {'L': 2, 'RGB': 6}.get(mode, -1)
    if kind == b'sBIT':
        return n == {'L': 1, 'P': 3, 'RGB': 3, 'RGBA': 4}[mode]
    if kind == b'bKGD':
        return n == {'L': 2, 'P': 1, 'RGB': 6, 'RGBA': 6}[mode]
    return kind == b'tEXt'


def parse(data) -> Optional[Header]:
    """The file's Header when it is device-eligible (see the module's docstring), else None."""
    from PIL import Image
    data = memoryview(data)
    if bytes(data[:8]) != SIGNATURE:
        return None
    chunks, pos, end = [], 8, len(data)
    while pos < end:
        if pos + 12 > end:
            return None
        n, kind = struct.unpack_from('>I4s', data, pos)
        stop = pos + 8 + n
        if n >= 1 << 31 or stop + 4 > end or zlib.crc32(data[pos + 4:stop]) != struct.unpack_from('>I', data, stop)[0]:
            return None
        chunks.append((kind, pos + 8, stop))
        pos = stop + 4
        if kind == b'IEND':
            break
    if pos != end or len(chunks) < 3 or chunks[0][0] != b'IHDR' or chunks[0][2] - chunks[0][1] != 13 or \
            chunks[-1][0] != b'IEND' or chunks[-1][2] != chunks[-1][1]:
        return None
    w, h, bits, colour_type, compression, filter_method, interlace = struct.unpack_from('>IIBBBBB', data, chunks[0][1])
    mode = _MODES.get((colour_type, bits))
    if mode is None or not (1 <= w < 1 << 31 and 1 <= h < 1 << 31) or compression or filter_method or interlace:
        return None
    if Image.MAX_IMAGE_PIXELS is not None and w * h > Image.MAX_IMAGE_PIXELS:
        return None
    idat = [k for k, c in enumerate(chunks) if c[0] == b'IDAT']
    if not idat or idat[-1] - idat[0] + 1 != len(idat):
        return None
    seen, text, palette_entries = set(), 0, 0
    for k, (kind, a, b) in enumerate(chunks[1:-1], 1):
        if kind == b'IDAT':
            continue
        before = k < idat[0]
        if kind == b'PLTE':
            if mode != 'P' or not before or kind in seen or (b - a) % 3 or not 3 <= b - a <= 768:
                return None
            palette_entries = (b - a) // 3
        elif kind not in ANCILLARY or not (before or kind in _AFTER_IDAT) or (kind in seen and kind != b'tEXt') or \
                not _ancillary_ok(kind, b - a, mode, palette_entries):
            return None
        text += (b - a) if kind == b'tEXt' else 0
        seen.add(kind)
    if (mode == 'P') != (b'PLTE' in seen) or text > TEXT_BYTES:
        return None
    return Header(h, w, colour_type, bits, mode, tuple((chunks[k][1], chunks[k][2]) for k in idat))


def _aligned(n):
    return (n + _ALIGN - 1) // _ALIGN * _ALIGN


def enqueue(files, device=None):
    """Enqueues one device launch for ``files``, a list of (file bytes, Header), on the current stream without
    synchronising the host.  -> (status int32 CUDA tensor [n], [CUDA uint8 tensor per file], keep): a file's tensor
    (a view of one buffer shared by the batch) holds Pillow's array once its status is 0; keep (the launch's device
    buffers) must stay referenced until the work completes."""
    from deva import _native
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    streams = [hd.stream(data) for data, hd in files]
    desc = np.zeros((len(files), _native.PNG_DESC_FIELDS), np.int64)
    s_at = out_at = work_at = 0
    for k, ((_, hd), st) in enumerate(zip(files, streams)):
        desc[k] = (s_at, len(st), hd.h, hd.w, hd.colour_type, hd.bits, out_at, work_at)
        s_at += len(st)
        out_at += _aligned(hd.nbytes)
        work_at += _native.png_decode_workspace_bytes(hd.h, hd.w, hd.colour_type, hd.bits)
    head = desc.nbytes
    host = torch.empty(head + s_at, dtype=torch.uint8, pin_memory=True)
    hnp = host.numpy()
    hnp[:head] = desc.reshape(-1).view(np.uint8)
    at = head
    for st in streams:
        hnp[at:at + len(st)] = np.frombuffer(st, np.uint8)
        at += len(st)
    dev = torch.empty(_aligned(head + s_at), dtype=torch.uint8, device=device)
    dev[:head + s_at].copy_(host, non_blocking=True)
    out = torch.empty(max(out_at, 1), dtype=torch.uint8, device=device)
    work = torch.empty(max(work_at, 1), dtype=torch.uint8, device=device)
    status = torch.empty(len(files), dtype=torch.int32, device=device)
    _native.png_decode(dev[head:head + s_at] if s_at else dev[head:head + 1], dev[:head].view(torch.int64).view(
        len(files), _native.PNG_DESC_FIELDS), out, work, status)
    arrays = [out[int(desc[k, 6]):int(desc[k, 6]) + hd.nbytes].view(hd.shape) for k, (_, hd) in enumerate(files)]
    return status, arrays, (dev, out, work)


def decode_batch(files, device=None):
    """One device launch for ``files``, a list of (file bytes, Header or None).  -> [(status, tensor)]: for a file
    with no Header (None, None); else the device's status and, when it is 0, the decoded CUDA uint8 tensor (a view of
    one buffer shared by the batch).  Synchronises the host once, to read the statuses."""
    todo = [(i, data, hd) for i, (data, hd) in enumerate(files) if hd is not None]
    results = [(None, None)] * len(files)
    if not todo:
        return results
    status, arrays, _ = enqueue([(data, hd) for _, data, hd in todo], device)
    for (i, _, _), st, t in zip(todo, status.tolist(), arrays):  # the batch's one synchronisation
        results[i] = (st, t if st == 0 else None)
    return results


read_bytes = device_decode.read_bytes


def batches(headers, budget=BUDGET):
    """Consecutive index ranges [a, b) of files whose decoded bytes (arrays and filtered streams) stay within budget;
    a file over the budget is a batch of its own.  headers: Header or None per file."""
    return device_decode.batches([0 if hd is None else 2 * hd.nbytes + hd.h for hd in headers], budget)


def decode_results(sources, device=None, budget=BUDGET, datas=None) -> List[object]:
    """Per source (a path or bytes), in order: the CUDA tensor of ``np.asarray(Image.open(source))``, or the exception
    Pillow raises for it.  datas: the sources' bytes when already read (None for an unreadable path)."""
    datas = [read_bytes(s) for s in sources] if datas is None else datas
    headers = [None if d is None else parse(d) for d in datas]
    costs = [0 if hd is None else 2 * hd.nbytes + hd.h for hd in headers]
    return device_decode.decode_results(sources, datas, headers, costs, decode_batch, device, budget)


def decode_pngs(sources) -> List[torch.Tensor]:
    """The CUDA tensors of ``np.asarray(Image.open(s))`` for every path or bytes ``s``; raises the first file's error
    that Pillow would raise."""
    return device_decode.raise_first(decode_results(sources))


def decode_png(source) -> torch.Tensor:
    """The CUDA tensor of ``np.asarray(Image.open(source))`` (a path or bytes); raises Pillow's error."""
    return decode_pngs([source])[0]
