"""The format-agnostic half of the device image decoders (deva/utils/png_decode.py, deva/utils/jpeg_decode.py): read
the sources, group the device-eligible files into batches under a budget of decoded bytes, decode each batch with one
synchronisation, and give every file the device's tensor or, where the device declined it, Pillow's array or Pillow's
exception.  Importing this module does not initialise CUDA."""
import io
from typing import Callable, List, Sequence

import numpy as np

from deva.utils import device_download


def read_bytes(source):
    """The bytes of a path or bytes source; None when a path cannot be read (Pillow then raises its own error)."""
    if isinstance(source, (bytes, bytearray, memoryview)):
        return bytes(source)
    try:
        with open(source, 'rb') as f:
            return f.read()
    except OSError:
        return None


def pillow_array(source) -> np.ndarray:
    """``np.asarray(Image.open(source))`` for a path or bytes source."""
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(source) if isinstance(source, (bytes, bytearray, memoryview)) else source))


def batches(costs: Sequence[int], budget: int):
    """Consecutive index ranges [a, b) of files whose costs stay within budget; a file over the budget is a batch of its
    own."""
    out, a, used = [], 0, 0
    for i, n in enumerate(costs):
        if i > a and used + n > budget:
            out.append((a, i))
            a, used = i, 0
        used += n
    if a < len(costs):
        out.append((a, len(costs)))
    return out


def decode_results(sources, datas, headers, costs, decode_batch: Callable, device, budget) -> List[object]:
    """Per source, in order: the device's CUDA tensor when ``decode_batch`` gave status 0 for it, else Pillow's array
    uploaded to the device, or the exception Pillow raises.  headers: the format's parse of each file (None: not
    device-eligible); decode_batch(list of (bytes, header)) -> [(status, tensor)]."""
    results = []
    for a, b in batches(costs, budget):
        for k, (st, t) in enumerate(decode_batch(list(zip(datas[a:b], headers[a:b])), device), a):
            if st == 0:
                results.append(t)
                continue
            try:
                arr = pillow_array(sources[k])
            except Exception as e:  # noqa: BLE001  (Pillow's own error is the result)
                results.append(e)
                continue
            up = device_download.upload(arr if arr.flags.writeable else arr.copy())  # Pillow's arrays are read-only
            results.append(up if device is None else up.to(device))
    return results


def raise_first(results):
    """results, unless one is an exception: then the first is raised."""
    for r in results:
        if isinstance(r, BaseException):
            raise r
    return results
