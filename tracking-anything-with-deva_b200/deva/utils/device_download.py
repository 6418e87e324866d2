"""The host side of the device encoders (deva/utils/png_encode.py, jpeg_encode.py, rle_encode.py): their option, their
upload and their download.

An encode writes one device buffer ``[header | payload | workspace]``.  The header is int64s, the last of them the
payload's length: the PNG stream's or JPEG scan's length, or the RLE strings' offsets.  The payload is at most ``bound``
bytes.  ``enqueue`` copies the header and the payload's first ``min(prefix, bound)`` bytes into the same bytes of a
pinned host buffer and records an event, on the current stream and without synchronising the host.
``Pending.result()`` waits for the event, fetches the rest of a longer payload, frees the device buffer and hands
header and payload to the encoder's finisher, which builds the file or the strings.  Importing this module does not
initialise CUDA.
"""
import os
from typing import Callable, List, Optional

import numpy as np
import torch


def resolve(value: Optional[str], option: str, env: str, choices, default: str) -> str:
    """``value``, or the environment's ``env`` when it is None (``default`` when that is unset); one of ``choices``."""
    value = os.environ.get(env, default) if value is None else value
    if value not in choices:
        raise ValueError(f'{option} must be one of {choices}, not {value!r}')
    return value


def upload(array: np.ndarray, dtype=None) -> torch.Tensor:
    """A contiguous CUDA copy of host ``array`` (as ``dtype`` when given), staged through pinned memory and copied
    without synchronising the host."""
    return torch.from_numpy(np.ascontiguousarray(array, dtype=dtype)).pin_memory().cuda(non_blocking=True)


def buffer(head: int, bound: int, workspace: int, device):
    """A device buffer ``[header | payload | workspace]`` of ``head`` header bytes, ``bound`` payload bytes and
    ``workspace`` bytes, the workspace 16-byte aligned as the encoders' C entry points require.  -> (buffer, payload
    view, workspace view)."""
    ws_at = (head + bound + 15) // 16 * 16
    dev = torch.empty(ws_at + workspace, dtype=torch.uint8, device=device)
    return dev, dev[head:head + bound], dev[ws_at:]


def pinned(host: Optional[torch.Tensor], nbytes: int) -> torch.Tensor:
    """``host``, a pinned uint8 buffer of at least ``nbytes`` bytes, or a new one when it is None."""
    if host is None:
        return torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    assert host.is_pinned() and host.dtype == torch.uint8 and host.numel() >= nbytes
    return host


class Pending:
    """An encode enqueued on the device; ``result()`` -> ``finish(header, payload)``, the encoder's file or strings."""

    def __init__(self, finish: Callable[[List[int], bytes], object], dev: Optional[torch.Tensor] = None,
                 host: Optional[torch.Tensor] = None, header=(0, 0), prefix: int = 0,
                 done: Optional[torch.cuda.Event] = None):
        self.finish, self.dev, self.host, self.header, self.prefix, self.done = finish, dev, host, header, prefix, done

    def result(self):
        header, payload = [], b''
        if self.done is not None:  # else nothing was encoded
            self.done.synchronize()
            start, at = self.header
            header = self.host[start:at].view(torch.int64).tolist()
            n = header[-1]
            payload = self.host[at:at + min(n, self.prefix)].numpy().tobytes()
            if n > self.prefix:
                payload += self.dev[at + self.prefix:at + n].cpu().numpy().tobytes()
            self.dev = None  # the device buffer is free once the payload is on the host
        return self.finish(header, payload)


def enqueue(finish, dev: torch.Tensor, header, bound: int, prefix: int, host: Optional[torch.Tensor]) -> Pending:
    """Copies ``dev``'s header, bytes ``header[0]:header[1]``, and the payload's first ``min(prefix, bound)`` bytes
    after it into the same bytes of the pinned buffer ``host`` (one is allocated when None), and records an event.
    ``host`` must stay untouched until ``result()`` returns."""
    start, at = header
    prefix = min(prefix, bound)
    host = pinned(host, at + prefix)
    host[start:at + prefix].copy_(dev[start:at + prefix], non_blocking=True)
    done = torch.cuda.Event()
    done.record()
    return Pending(finish, dev, host, header, prefix, done)


def write(pending: Pending, file: str):
    """Writes the file of an enqueued encode; waits for it."""
    data = pending.result()
    with open(file, 'wb') as f:
        f.write(data)
