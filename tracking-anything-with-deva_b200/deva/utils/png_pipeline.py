"""Host side of the per-video PNG passes (VIPSeg metrics, unsupervised DAVIS post-processing): PNGs decoded on a pool of
host threads, in order and ahead of use, and uint8 arrays uploaded through a ring of pinned staging slots.  Importing
this module does not initialise CUDA."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

RING = 4  # pinned staging slots: a slot is refilled only after its previous upload has completed


class Uploader:
    """uint8 host arrays -> device tensors on the current stream, through pinned slots; never synchronises the device."""

    def __init__(self, device):
        self.device = device
        self.slots = [None] * RING
        self.i = 0

    def __call__(self, a: np.ndarray) -> torch.Tensor:
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
