"""PNG files encoded on the device (``deva_b200_png_encode``): an opt-in replacement for Pillow's PNG writer in the
result saver and the post-processing passes, selected by ``png_encoder='device'`` or ``DEVA_B200_PNG_ENCODER=device``.

The format is fixed, so that oracle/png_encode.py restates it byte for byte.  It decodes (Pillow, zlib) to the pixels,
mode and palette of Pillow's own write of the same image; the bytes are not Pillow's, and the files are larger
(1.5-3.5x on segmentation maps, about 1 % of the raw bytes):
  * chunks: the PNG signature, IHDR, PLTE (P images only), one IDAT, IEND; every CRC-32 is the standard one;
  * colour type and bit depth follow Pillow's writer: L and RGB are 8-bit; a P image whose palette has <= 2 / 4 / 16
    colours is written at 1 / 2 / 4 bits, else 8, and PLTE holds the first ``colors * 3`` bytes of its palette.  A
    sub-byte row packs its pixels MSB-first with zero padding: ``v & (2^bits - 1)`` at 2 and 4 bits, ``v != 0`` at 1
    bit (what Pillow's packers store);
  * every row uses filter type 2 (Up; row 0 against zeros); the filtered stream ``s`` is the rows' ``[2] + filtered
    row bytes`` concatenated;
  * each row segment of ``s`` is tokenised on its own, greedily: at position i the candidate distances are 1 and bpp
    (bytes per complete pixel, at least 1), a candidate's length is the run of ``s[j] == s[j - d]`` with ``j - d >= 0``
    in stream coordinates and ``j`` inside the row segment, capped at 258; the longer candidate wins, a tie takes the
    smaller distance; a length >= 3 is a match, anything shorter the literal ``s[i]``;
  * one deflate block, BFINAL = 1, BTYPE = 01 (RFC 1951's fixed codes): the tokens in order, end-of-block, zero padding;
  * zlib header 0x78 0x01 and the big-endian Adler-32 of ``s``.
Every literal takes at most 9 bits, which bounds the stream at ``ceil((3 + 9 len(s) + 7) / 8) + 6`` bytes.

The device writes the zlib stream and its length; the chunks and their CRCs are built here around the downloaded
stream.  ``encode_png_async`` enqueues the encode and a copy of the stream's first ``PREFIX`` bytes on the current
stream without synchronising, and the returned ``Pending``'s ``result()`` waits for them (and fetches the rest of a
larger stream; deva/utils/device_download.py).  Importing this module does not initialise CUDA.
"""
import functools
import struct
import zlib
from typing import Optional

import numpy as np
import torch

from deva.utils import device_download

ENCODERS = ('pil', 'device')
ENV = 'DEVA_B200_PNG_ENCODER'
PREFIX = 128 * 1024  # stream bytes copied with the encode; a longer stream's remainder is fetched by result()
SIGNATURE = b'\x89PNG\r\n\x1a\n'
_COLOUR_TYPE = {'L': 0, 'RGB': 2, 'P': 3}


def resolve_encoder(png_encoder: Optional[str] = None) -> str:
    """``png_encoder``, or the environment's ``DEVA_B200_PNG_ENCODER`` when it is None ('pil' when that is unset)."""
    return device_download.resolve(png_encoder, 'png_encoder', ENV, ENCODERS, 'pil')


@functools.lru_cache(maxsize=64)
def _palette_layout(palette):
    from PIL import Image
    im = Image.new('P', (1, 1))
    if palette is not None:
        im.putpalette(palette)
    colors = max(min(len(im.palette.getdata()[1]) // 3, 256), 1) if im.palette else 256
    bits = 1 if colors <= 2 else 2 if colors <= 4 else 4 if colors <= 16 else 8
    plte = im.im.getpalette('RGB')[:colors * 3]
    return bits, plte + b'\0' * (colors * 3 - len(plte))


def pillow_png_layout(mode: str, palette=None):
    """(bit depth, PLTE bytes or None) of Pillow's PNG writer for an image of ``mode`` ('L', 'RGB' or 'P') whose palette
    was set with ``putpalette(palette)``."""
    if mode not in _COLOUR_TYPE:
        raise ValueError(f'mode must be L, RGB or P, not {mode!r}')
    if mode != 'P':
        return 8, None
    return _palette_layout(None if palette is None else bytes(palette))


def _chunk(kind: bytes, data: bytes) -> bytes:
    return struct.pack('>I', len(data)) + kind + data + struct.pack('>I', zlib.crc32(kind + data))


def host_bytes() -> int:
    """Bytes of the pinned buffer ``encode_png_async`` needs: the stream's length and its first ``PREFIX`` bytes."""
    return 8 + PREFIX


def _as_device_image(img, mode):
    if isinstance(img, np.ndarray):
        img = device_download.upload(img)
    want = 3 if mode == 'RGB' else 2
    if not (img.is_cuda and img.dtype == torch.uint8 and img.dim() == want and (mode != 'RGB' or img.shape[2] == 3)):
        raise ValueError(f'a {mode} image is a CUDA uint8 tensor [h, w{", 3" if mode == "RGB" else ""}], not '
                         f'{img.dtype} {tuple(img.shape)} on {img.device}')
    return img.contiguous()


def encode_png_async(img, mode: str, palette=None, host: Optional[torch.Tensor] = None) -> device_download.Pending:
    """Enqueues the encode of uint8 ``img`` ([h, w] for 'L' / 'P', [h, w, 3] for 'RGB'; a CUDA tensor, or a numpy
    array that is uploaded) on the current stream; never synchronises the host.  host: optional pinned uint8 buffer of
    at least ``host_bytes()`` bytes that receives the stream's length and first bytes (one is allocated otherwise); it
    must stay untouched until ``result()`` returns, which gives the PNG file's bytes."""
    from deva import _native
    bits, plte = pillow_png_layout(mode, palette)
    img = _as_device_image(img, mode)
    h, w = img.shape[:2]
    channels = 3 if mode == 'RGB' else 1
    bound = _native.png_bound(h, w, channels, bits)
    dev, out, ws = device_download.buffer(8, bound, _native.png_workspace_bytes(h), img.device)
    _native.png_encode(img, bits, ws, out, dev[:8].view(torch.int64))
    head = SIGNATURE + _chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, bits, _COLOUR_TYPE[mode], 0, 0, 0))
    if plte is not None:
        head += _chunk(b'PLTE', plte)
    return device_download.enqueue(lambda _, idat: head + _chunk(b'IDAT', idat) + _chunk(b'IEND', b''), dev, (0, 8),
                                   bound, PREFIX, host)


def encode_png(img, mode: str, palette=None) -> bytes:
    """The PNG file of uint8 ``img`` (see ``encode_png_async``); waits for the device."""
    return encode_png_async(img, mode, palette).result()
