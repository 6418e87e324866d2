"""Host side of the per-video PNG passes (VIPSeg metrics, unsupervised DAVIS post-processing): PNGs decoded on a pool of
host threads, in order and ahead of use, and uint8 arrays uploaded through a ring of pinned staging slots; or, with
``png_decoder='device'``, file bytes read on the pool and decoded a video at a time on the device (DeviceDecoder).
Importing this module does not initialise CUDA."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from deva.utils import png_decode

RING = 4  # pinned staging slots: a slot is refilled only after its previous upload has completed


class Uploader:
    """uint8 host arrays -> device tensors on the current stream, through pinned slots; never synchronises the device.
    A frame already on the device (from DeviceDecoder) is returned as it is."""

    def __init__(self, device):
        self.device = device
        self.slots = [None] * RING
        self.i = 0

    def __call__(self, a: np.ndarray) -> torch.Tensor:
        if isinstance(a, torch.Tensor):
            return a
        k = self.i % RING
        self.i += 1
        n = a.size
        slot = self.slots[k]
        if slot is None or slot[0].numel() < n:
            slot = (torch.empty(n, dtype=torch.uint8, pin_memory=True), torch.cuda.Event())
            self.slots[k] = slot
        host, done = slot
        done.synchronize()
        host[:n].numpy()[:] = a.reshape(-1)  # PIL's arrays are read-only: numpy copies without wrapping them
        dev = torch.empty(a.shape, dtype=torch.uint8, device=self.device)
        dev.view(-1).copy_(host[:n], non_blocking=True)
        done.record()
        return dev


class Decoder:
    """A pool of host threads decoding files with ``read(path)``; ``frames(paths)`` yields the results in order while
    later ones decode."""

    def __init__(self, read, num_threads=None):
        self.read = read
        self.pool = ThreadPoolExecutor(max_workers=num_threads or min(16, os.cpu_count() or 1))

    def frames(self, paths):
        return self.pool.map(self.read, paths)

    def close(self):
        self.pool.shutdown()


class DeviceDecoder(Decoder):
    """Files read and parsed on the pool and decoded on the device (deva/utils/png_decode.py), one ``frames`` call (a
    video) in batches of at most ``png_decode.BUDGET`` decoded bytes; a batch is decoded when its first frame is
    reached.  A frame is a CUDA tensor when the device decoded it; a file the device does not take (ineligible, refused
    by the device, or of a mode outside ``modes``) is read by ``read(path)`` on the pool as Decoder reads it, so its
    array, its error marker and the exception it raises are Decoder's.  rgb: RGBA frames are sliced to their RGB
    channels on the device, as read_rgb does on the host.  A frame is a view of its batch's output buffer, which stays
    allocated while any of the batch's frames is held."""

    def __init__(self, read, device, modes=('L', 'P', 'RGB', 'RGBA'), rgb=False, num_threads=None):
        super().__init__(read, num_threads)
        self.device, self.modes, self.rgb = device, modes, rgb

    def _parsed(self, path):
        data = png_decode.read_bytes(path)
        header = None if data is None else png_decode.parse(data)
        return data, header if header is not None and header.mode in self.modes else None

    def frames(self, paths):
        parsed = [self.pool.submit(self._parsed, p) for p in paths]  # ahead of use, like Decoder.frames
        return self._frames(paths, parsed)

    def _frames(self, paths, parsed):
        files = [p.result() for p in parsed]
        for a, b in png_decode.batches([h for _, h in files]):
            frames = []
            for status, t in png_decode.decode_batch(files[a:b], self.device):
                if status == 0 and self.rgb and t.dim() == 3 and t.shape[2] == 4:
                    t = t[:, :, :3].contiguous()
                frames.append(t if status == 0 else None)
            rest = {k: self.pool.submit(self.read, paths[a + k]) for k, f in enumerate(frames) if f is None}
            for k, f in enumerate(frames):
                yield rest[k].result() if k in rest else f
