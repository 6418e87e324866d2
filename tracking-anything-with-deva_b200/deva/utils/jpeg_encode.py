"""Baseline JPEG files encoded on the device (``deva_b200_jpeg_encode``): an opt-in replacement for Pillow's JPEG writer in
the result saver, selected by ``jpeg_encoder='device'`` or ``DEVA_B200_JPEG_ENCODER=device``.

The file is byte for byte what Pillow's default ``Image.fromarray(rgb).save(f, 'JPEG', quality=q)`` writes through
libjpeg(-turbo), because every step is libjpeg's integer arithmetic (oracle/jpeg_encode.py restates it):
  * RGB -> YCbCr in jccolor.c's 16-bit fixed point; 4:2:0 downsampling ``(a + b + c + d + bias) >> 2`` with bias
    1, 2, 1, 2, ...; the last column replicated, the input padded to an even row count and the downsampled planes by
    repeating their last row;
  * level shift, the ``islow`` integer DCT, rounding quantisation with the Annex K tables scaled for ``quality`` (as
    ``jpeg_set_quality(q, force_baseline=True)``);
  * MCU order Y00 Y01 Y10 Y11 Cb Cr, libjpeg's dummy blocks at the right and bottom edges, the Annex K Huffman tables,
    a 1-bit fill and a 0x00 stuffed after every 0xFF;
  * markers SOI, APP0 (JFIF 1.01, no units, density 1x1), DQT 0, DQT 1, SOF0, DHT DC0 AC0 DC1 AC1, SOS, scan, EOI.

The device writes the scan, EOI and its length; the marker segments are built here.  ``encode_jpeg_async`` enqueues
the encode and a copy of the scan's first ``PREFIX`` bytes on the current stream without synchronising, and the
returned ``Pending``'s ``result()`` waits for them (and fetches the rest of a longer scan;
deva/utils/device_download.py).  Importing this module does not initialise CUDA.
"""
import functools
import struct
from typing import Optional

import numpy as np
import torch

from deva.utils import device_download

ENCODERS = ('pil', 'device')
ENV = 'DEVA_B200_JPEG_ENCODER'
PREFIX = 1024 * 1024  # scan bytes copied with the encode (a 1080p overlay's whole scan); result() fetches the rest
MAX_SIDE = 65535

# Annex K.1 quantisation tables, natural order
_LUMA_Q = (16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
           14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
           49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99)
_CHROMA_Q = (17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
             47, 66, 99, 99, 99, 99, 99, 99) + (99, ) * 32
_ZIGZAG = (0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
           21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
           60, 61, 54, 47, 55, 62, 63)
# Annex K.3 Huffman tables: code counts per length 1..16, then the symbols
_DHT = (
    (0x00, bytes([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0]) + bytes(range(12))),
    (0x10, bytes([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d]) + bytes.fromhex(
        '01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738'
        '393a434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4'
        'a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa')),
    (0x01, bytes([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0]) + bytes(range(12))),
    (0x11, bytes([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77]) + bytes.fromhex(
        '000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a3536'
        '3738393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999a'
        'a2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa')),
)


def resolve_encoder(jpeg_encoder: Optional[str] = None) -> str:
    """``jpeg_encoder``, or the environment's ``DEVA_B200_JPEG_ENCODER`` when it is None ('pil' when that is unset)."""
    return device_download.resolve(jpeg_encoder, 'jpeg_encoder', ENV, ENCODERS, 'pil')


@functools.lru_cache(maxsize=128)
def quant_tables(quality: int = 75) -> bytes:
    """Luma then chroma quantisation tables (64 bytes each, zigzag order) of ``jpeg_set_quality(quality, True)``."""
    if not (isinstance(quality, (int, np.integer)) and 1 <= quality <= 100):
        raise ValueError(f'quality must be an integer in [1, 100], not {quality!r}')
    scale = 5000 // quality if quality < 50 else 200 - 2 * quality
    return bytes(min(max((base[k] * scale + 50) // 100, 1), 255) for base in (_LUMA_Q, _CHROMA_Q) for k in _ZIGZAG)


def _segment(marker: int, body: bytes) -> bytes:
    return struct.pack('>BBH', 0xff, marker, len(body) + 2) + body


@functools.lru_cache(maxsize=64)
def headers(h: int, w: int, quality: int = 75) -> bytes:
    """The marker segments before the scan: SOI, APP0, DQT 0, DQT 1, SOF0, the four DHTs and SOS."""
    tables = quant_tables(quality)
    out = b'\xff\xd8' + _segment(0xe0, b'JFIF\0' + bytes([1, 1, 0]) + struct.pack('>HHBB', 1, 1, 0, 0))
    out += _segment(0xdb, b'\0' + tables[:64]) + _segment(0xdb, b'\1' + tables[64:])
    out += _segment(0xc0, struct.pack('>BHHB', 8, h, w, 3) + bytes([1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for tc_th, body in _DHT:
        out += _segment(0xc4, bytes([tc_th]) + body)
    return out + _segment(0xda, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))


def host_bytes() -> int:
    """Bytes of the pinned buffer ``encode_jpeg_async`` needs: the scan's length and its first ``PREFIX`` bytes."""
    return 8 + PREFIX


def _as_device_image(img):
    if isinstance(img, np.ndarray):
        if not (img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3):
            raise ValueError(f'a JPEG image is uint8 RGB [h, w, 3], not {img.dtype} {img.shape}')
        _check_sides(img.shape)
        return device_download.upload(img)
    if not (isinstance(img, torch.Tensor) and img.is_cuda and img.dtype == torch.uint8 and img.dim() == 3 and
            img.shape[2] == 3):
        desc = f'{img.dtype} {tuple(img.shape)} on {img.device}' if isinstance(img, torch.Tensor) else type(img)
        raise ValueError(f'a JPEG image is a CUDA uint8 RGB tensor [h, w, 3] or a numpy array, not {desc}')
    _check_sides(img.shape)
    return img.contiguous()


def _check_sides(shape):
    if not (1 <= shape[0] <= MAX_SIDE and 1 <= shape[1] <= MAX_SIDE):
        raise ValueError(f'a JPEG image has sides in [1, {MAX_SIDE}], not {shape[0]} x {shape[1]}')


def encode_jpeg_async(img, quality: int = 75, host: Optional[torch.Tensor] = None) -> device_download.Pending:
    """Enqueues the encode of uint8 RGB ``img`` [h, w, 3] (a CUDA tensor, or a numpy array that is uploaded) on the
    current stream; never synchronises the host.  host: optional pinned uint8 buffer of at least ``host_bytes()`` bytes
    that receives the scan's length and first bytes (one is allocated otherwise); it must stay untouched until
    ``result()`` returns, which gives the JPEG file's bytes."""
    from deva import _native
    tables = quant_tables(quality)
    img = _as_device_image(img)
    h, w = img.shape[:2]
    bound = _native.jpeg_bound(h, w)
    dev, out, ws = device_download.buffer(8, bound, _native.jpeg_workspace_bytes(h, w), img.device)
    _native.jpeg_encode(img, tables, ws, out, dev[:8].view(torch.int64))
    head = headers(h, w, quality)
    return device_download.enqueue(lambda _, scan: head + scan, dev, (0, 8), bound, PREFIX, host)


def encode_jpeg(img, quality: int = 75) -> bytes:
    """The JPEG file of uint8 RGB ``img`` (see ``encode_jpeg_async``); waits for the device."""
    return encode_jpeg_async(img, quality).result()
