"""Baseline JPEG files decoded on the device (``deva_b200_jpeg_decode``): an opt-in replacement for Pillow's JPEG
reader, selected by ``jpeg_decoder='device'`` or ``DEVA_B200_JPEG_DECODER=device``.

For every file the result is exactly what Pillow gives: ``np.asarray(Image.open(f))`` as a CUDA tensor, or the
exception Pillow raises.  The device takes the plain, well-formed case and every other file is read by Pillow, so none of
libjpeg's recovery from corrupt data (warnings, zero-filled MCUs, resynchronisation) is restated here.  A file is
device-eligible (``parse``, decided on the host) when:
  * it starts with SOI and ends with EOI as its last two bytes, with no fill bytes between markers;
  * before the scan there are only APPn, COM, DQT with 8-bit tables, DHT that libjpeg accepts (at most 256 symbols,
    no code overflow, DC symbols <= 15), DRI, one SOF0 and one SOS;
  * SOF0 has 8-bit precision, 1 <= w, h <= 65535, ``w * h <= Image.MAX_IMAGE_PIXELS``, three components with distinct
    ids, Y sampled 1x1, 2x1 or 2x2 and Cb, Cr 1x1;
  * SOS names the three components in SOF order with defined tables, Ss = 0, Se = 63, Ah = Al = 0;
  * the scan holds no marker other than RSTn in sequence, exactly one per restart interval boundary, and every
    interval has data;
  * libjpeg-turbo would take the components as YCbCr and Pillow reads no APPn payload that could raise: no Adobe APP14,
    no Exif APP1, no ICC_PROFILE, FPXR or MPF APP2, no JFIF APP0 shorter than 14 bytes, and component ids other than
    'R', 'G', 'B'.
The host removes the stuffing bytes and RSTn markers and cuts each restart interval into ``SUB_BYTES``-byte
subsequences; the device decodes them in parallel (csrc/jpeg_decode.cu) and gives a nonzero status, which sends the file
to Pillow, for a code not in the table, a category over 11 (DC) or 10 (AC), a run past coefficient 63, an interval that
ends early or has data after its last MCU, or a block outside the range where libjpeg-turbo's C and x86 SIMD islow IDCTs
agree.

Importing this module does not initialise CUDA.
"""
import struct
from typing import List, NamedTuple, Optional

import numpy as np
import torch

from deva.utils import device_decode, device_download

DECODERS = ('pil', 'device')
ENV = 'DEVA_B200_JPEG_DECODER'
BUDGET = 256 << 20   # decoded bytes (arrays, sample planes and coefficients) of one batch
SUB_BYTES = 128      # bytes of the compacted scan per subsequence
DESC_FIELDS = 11
IV_FIELDS = 6
SUB_FIELDS = 3
HUFF_WORDS = 512 + 18 + 18 + 256
TABLE_WORDS = 6 * HUFF_WORDS + 3 * 64
_ALIGN = 16
# jpeg_natural_order: the natural index of the k-th zig-zag coefficient
NATURAL = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                    6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                    38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])


class Header(NamedTuple):
    """A device-eligible file: its shape, luma sampling, tables (int32 [TABLE_WORDS]), the scan without stuffing
    bytes and RSTn markers, and its restart intervals as (byte start, byte end, first MCU, MCUs)."""
    h: int
    w: int
    hy: int
    vy: int
    tables: np.ndarray
    scan: np.ndarray
    intervals: tuple

    @property
    def shape(self):
        return (self.h, self.w, 3)

    @property
    def nbytes(self):
        return self.h * self.w * 3

    @property
    def mcus(self):
        return ((self.w + 8 * self.hy - 1) // (8 * self.hy)) * ((self.h + 8 * self.vy - 1) // (8 * self.vy))

    @property
    def blocks(self):
        return self.mcus * (self.hy * self.vy + 2)

    @property
    def cost(self):
        """Device bytes of the decode: the array, the sample planes, the coefficients and the subsequences' state."""
        subs = sum(-(-(b - a) // SUB_BYTES) for a, b, _, _ in self.intervals)
        return self.nbytes + self.blocks * (64 + 128) + subs * 120  # two exits, an entry and a prefix


def resolve_decoder(jpeg_decoder: Optional[str] = None) -> str:
    """``jpeg_decoder``, or the environment's ``DEVA_B200_JPEG_DECODER`` when it is None ('pil' when that is unset)."""
    return device_download.resolve(jpeg_decoder, 'jpeg_decoder', ENV, DECODERS, 'pil')


def huff_table(bits, vals, dc):
    """int32 [HUFF_WORDS] lookup of a DHT table (bits: 16 code counts, vals: symbols), or None when libjpeg's
    jpeg_make_d_derived_tbl would refuse it."""
    fast = np.zeros(512, np.int32)
    maxcode = np.full(18, -1, np.int32)
    valoff = np.zeros(18, np.int32)
    code, p = 0, 0
    for length in range(1, 17):
        n = bits[length - 1]
        if n:
            valoff[length] = p - code
            for _ in range(n):
                if length <= 9:
                    lo = code << (9 - length)
                    fast[lo:lo + (1 << (9 - length))] = length << 8 | vals[p]
                code += 1
                p += 1
            maxcode[length] = code - 1
        if code >= 1 << length:
            return None
        code <<= 1
    if dc and any(v > 15 for v in vals):
        return None
    out = np.zeros(HUFF_WORDS, np.int32)
    out[:512] = fast
    out[512:530] = maxcode
    out[530:548] = valoff
    out[548:548 + len(vals)] = vals
    return out


def _app_ok(marker, seg):
    n = marker & 15
    if n == 0 and seg[:4] == b'JFIF':
        return len(seg) >= 14
    if n == 1 and seg[:6] == b'Exif\0\0':
        return False
    if n == 2 and (seg[:12] == b'ICC_PROFILE\0' or seg[:5] == b'FPXR\0' or seg[:4] == b'MPF\0'):
        return False
    return not (n == 14 and seg[:5] == b'Adobe')


def parse(data) -> Optional[Header]:
    """The file's Header when it is device-eligible (see the module's docstring), else None."""
    from PIL import Image
    data = bytes(data)
    end = len(data)
    if data[:2] != b'\xff\xd8' or end < 4 or data[-2:] != b'\xff\xd9':
        return None
    pos, quant, huff, restart, sof, sos = 2, {}, {}, 0, None, None
    while sos is None:
        if pos + 4 > end or data[pos] != 0xFF:
            return None
        marker, length = data[pos + 1], struct.unpack_from('>H', data, pos + 2)[0]
        seg, pos = data[pos + 4:pos + 2 + length], pos + 2 + length
        if length < 2 or pos > end:
            return None
        if 0xE0 <= marker <= 0xEF:
            if not _app_ok(marker, seg):
                return None
        elif marker == 0xFE:
            pass
        elif marker == 0xDB:
            while seg:
                if seg[0] >> 4 or seg[0] > 3 or len(seg) < 65:
                    return None
                q = np.zeros(64, np.int32)
                q[NATURAL] = np.frombuffer(seg[1:65], np.uint8)
                quant[seg[0]] = q
                seg = seg[65:]
        elif marker == 0xC4:
            while seg:
                if len(seg) < 17 or seg[0] & 0xEF > 3:
                    return None
                bits = list(seg[1:17])
                count = sum(bits)
                if count > 256 or len(seg) < 17 + count:
                    return None
                huff[seg[0] >> 4, seg[0] & 15] = (bits, list(seg[17:17 + count]))
                seg = seg[17 + count:]
        elif marker == 0xDD:
            if length != 4:
                return None
            restart = struct.unpack('>H', seg)[0]
        elif marker == 0xC0:
            if sof is not None or length != 17 or seg[0] != 8 or seg[5] != 3:
                return None
            sof = seg
        elif marker == 0xDA:
            if sof is None or length != 12 or seg[0] != 3 or seg[7:10] != b'\x00\x3f\x00':
                return None
            sos = seg
        else:
            return None
    h, w = struct.unpack_from('>HH', sof, 1)
    ids = [sof[6 + 3 * c] for c in range(3)]
    samp = [(sof[7 + 3 * c] >> 4, sof[7 + 3 * c] & 15) for c in range(3)]
    tq = [sof[8 + 3 * c] for c in range(3)]
    if h < 1 or w < 1 or len(set(ids)) != 3 or ids == [82, 71, 66] or samp[0] not in ((1, 1), (2, 1), (2, 2)) or \
            samp[1] != (1, 1) or samp[2] != (1, 1) or any(t not in quant for t in tq):
        return None
    if Image.MAX_IMAGE_PIXELS is not None and w * h > Image.MAX_IMAGE_PIXELS:
        return None
    tables = np.zeros(TABLE_WORDS, np.int32)
    for c in range(3):
        if sos[1 + 2 * c] != ids[c]:
            return None
        for k, key in enumerate(((0, sos[2 + 2 * c] >> 4), (1, sos[2 + 2 * c] & 15))):
            if key not in huff:
                return None
            t = huff_table(*huff[key], dc=k == 0)
            if t is None:
                return None
            tables[(2 * c + k) * HUFF_WORDS:(2 * c + k + 1) * HUFF_WORDS] = t
        tables[6 * HUFF_WORDS + 64 * c:6 * HUFF_WORDS + 64 * (c + 1)] = quant[tq[c]]
    hy, vy = samp[0]
    scan = np.frombuffer(data, np.uint8, end - 2 - pos, pos)
    ff = np.flatnonzero(scan == 0xFF)
    if len(ff) and ff[-1] == len(scan) - 1:
        return None
    nxt = scan[ff + 1]
    rst = (nxt & 0xF8) == 0xD0
    if not np.all((nxt == 0) | rst):
        return None
    at = ff[rst]
    if np.any(nxt[rst] != 0xD0 + np.arange(len(at)) % 8):
        return None
    mcus = ((w + 8 * hy - 1) // (8 * hy)) * ((h + 8 * vy - 1) // (8 * vy))
    n_iv = (mcus + restart - 1) // restart if restart else 1
    if len(at) != n_iv - 1:
        return None
    removed = np.sort(np.concatenate([ff[~rst] + 1, at, at + 1]))  # stuffing bytes and RSTn markers
    # an interval ends where its RSTn starts: that position less the bytes removed before it
    bounds = [0] + [int(a) - int(np.searchsorted(removed, a)) for a in at] + [len(scan) - len(removed)]
    per = restart if restart else mcus
    intervals = tuple((bounds[k], bounds[k + 1], k * per, min(per, mcus - k * per)) for k in range(n_iv))
    if any(a == b for a, b, _, _ in intervals):
        return None
    return Header(h, w, hy, vy, tables, np.delete(scan, removed), intervals)


def _aligned(n):
    return (n + _ALIGN - 1) // _ALIGN * _ALIGN


def layout(headers, sub_bytes=SUB_BYTES):
    """The batch's host records for ``headers``: (desc int64 [n, DESC_FIELDS], intervals int64 [., IV_FIELDS], subs
    int64 [., SUB_FIELDS], tables int32 [n, TABLE_WORDS], scans uint8, output bytes, workspace bytes)."""
    from deva import _native
    n = len(headers)
    desc = np.zeros((n, DESC_FIELDS), np.int64)
    ivs, subs = [], []
    scan_at = out_at = 0
    work_at = 0
    for f, hd in enumerate(headers):
        first_sub = sum(len(s) for s in subs)
        f_subs = []
        bpm = hd.hy * hd.vy + 2
        for a, b, m0, m in hd.intervals:
            starts = np.arange(a, b, sub_bytes, dtype=np.int64)
            stops = np.minimum(starts + sub_bytes, b)
            rows = np.stack([np.full(len(starts), len(ivs), np.int64), (scan_at + starts) * 8, (scan_at + stops) * 8],
                            1)
            ivs.append((f, (scan_at + a) * 8, (scan_at + b) * 8, m0 * bpm, m * bpm, first_sub + sum(map(len, f_subs))))
            f_subs.append(rows)
        subs.extend(f_subs)
        n_subs = sum(len(s) for s in f_subs)
        desc[f] = (scan_at, len(hd.scan), hd.h, hd.w, hd.hy, hd.vy, f, out_at, work_at, first_sub, n_subs)
        scan_at += len(hd.scan)
        out_at += _aligned(hd.nbytes)
        work_at += _native.jpeg_decode_workspace_bytes(hd.h, hd.w, hd.hy, hd.vy, n_subs)
    tables = np.stack([hd.tables for hd in headers]) if n else np.zeros((0, TABLE_WORDS), np.int32)
    scans = np.concatenate([hd.scan for hd in headers]) if n else np.zeros(0, np.uint8)
    sub_arr = np.concatenate(subs) if subs else np.zeros((0, SUB_FIELDS), np.int64)
    return (desc, np.array(ivs, np.int64).reshape(-1, IV_FIELDS), sub_arr, tables, scans, out_at,
            _native.jpeg_decode_workspace_bytes(0, 0, 0, 0, 0) + work_at)


def stage(headers, device=None, sub_bytes=SUB_BYTES):
    """Uploads the batch's records through one pinned copy and allocates its output and workspace, without
    synchronising.  -> (the device arguments of ``_native.jpeg_decode``, [CUDA uint8 tensor [h, w, 3] per file])."""
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    if device != torch.device('cuda', torch.cuda.current_device()):
        raise ValueError(f'jpeg_decode: the decode runs on the current device, not {device}')
    desc, ivs, subs, tables, scans, out_bytes, work_bytes = layout(headers, sub_bytes)
    parts = [desc.reshape(-1).view(np.uint8), ivs.reshape(-1).view(np.uint8), subs.reshape(-1).view(np.uint8),
             tables.reshape(-1).view(np.uint8), scans]
    offs, at = [], 0
    for p in parts:
        offs.append(at)
        at = _aligned(at + len(p))
    host = torch.empty(max(at, 1), dtype=torch.uint8, pin_memory=True)
    hnp = host.numpy()
    for o, p in zip(offs, parts):
        hnp[o:o + len(p)] = p
    dev = torch.empty(max(at, 1), dtype=torch.uint8, device=device)
    dev.copy_(host, non_blocking=True)

    def view(k, dtype, shape):
        return dev[offs[k]:offs[k] + max(len(parts[k]), 1)].view(dtype)[:int(np.prod(shape))].view(shape)
    out = torch.empty(max(out_bytes, 1), dtype=torch.uint8, device=device)
    work = torch.empty(work_bytes, dtype=torch.uint8, device=device)
    status = torch.empty(len(headers), dtype=torch.int32, device=device)
    args = (view(4, torch.uint8, (len(scans),)), view(0, torch.int64, desc.shape), view(3, torch.int32, tables.shape),
            view(1, torch.int64, ivs.shape), view(2, torch.int64, subs.shape), out, work, status)
    return args, [out[int(desc[k, 7]):int(desc[k, 7]) + hd.nbytes].view(hd.shape) for k, hd in enumerate(headers)]


def sync_rounds(args) -> int:
    """The synchronisation rounds the last decode with these arguments took (reads the device: synchronises)."""
    return int(args[6][:16].view(torch.int32)[3].item())


def enqueue(headers, device=None, sub_bytes=SUB_BYTES):
    """Enqueues the decode of ``headers`` on the current stream without synchronising the host.  -> (status int32
    CUDA tensor [n], [CUDA uint8 tensor [h, w, 3] per file], args): a file's tensor holds Pillow's array once its status
    is 0; args (the launch's device buffers) must stay referenced until the work completes."""
    from deva import _native
    args, arrays = stage(headers, device, sub_bytes)
    _native.jpeg_decode(*args)
    return args[7], arrays, args


def decode_batch(files, device=None):
    """One device launch for ``files``, a list of (file bytes, Header or None).  -> [(status, tensor)]: for a file
    with no Header (None, None); else the device's status and, when it is 0, the decoded CUDA uint8 tensor (a view of
    one buffer shared by the batch).  Synchronises the host once, to read the statuses."""
    todo = [(i, hd) for i, (_, hd) in enumerate(files) if hd is not None]
    results = [(None, None)] * len(files)
    if not todo:
        return results
    status, arrays, _ = enqueue([hd for _, hd in todo], device)
    for (i, _), st, t in zip(todo, status.tolist(), arrays):  # the batch's one synchronisation
        results[i] = (st, t if st == 0 else None)
    return results


def decode_results(sources, device=None, budget=BUDGET, datas=None) -> List[object]:
    """Per source (a path or bytes), in order: the CUDA tensor of ``np.asarray(Image.open(source))``, or the exception
    Pillow raises for it.  datas: the sources' bytes when already read (None for an unreadable path)."""
    datas = [device_decode.read_bytes(s) for s in sources] if datas is None else datas
    headers = [None if d is None else parse(d) for d in datas]
    costs = [0 if hd is None else hd.cost for hd in headers]
    return device_decode.decode_results(sources, datas, headers, costs, decode_batch, device, budget)


def decode_jpegs(sources) -> List[torch.Tensor]:
    """The CUDA tensors of ``np.asarray(Image.open(s))`` for every path or bytes ``s``; raises the first file's error
    that Pillow would raise."""
    return device_decode.raise_first(decode_results(sources))


def decode_jpeg(source) -> torch.Tensor:
    """The CUDA tensor of ``np.asarray(Image.open(source))`` (a path or bytes); raises Pillow's error."""
    return decode_jpegs([source])[0]


def decode_async(header: Header):
    """Enqueues one parsed file's decode on the current stream without synchronising.  -> (frame, status, keep):
    frame a CUDA uint8 [h, w, 3] tensor that holds Pillow's array when the int32 CUDA tensor status [1] reads 0; keep
    must stay referenced until the stream has passed the decode."""
    status, arrays, work = enqueue([header])
    return arrays[0], status, work
