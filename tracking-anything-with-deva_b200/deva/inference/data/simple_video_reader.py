"""``SimpleVideoReader``: the demos' frame reader, item for item what the reference's gives - ``(np.array(
Image.open(p).convert('RGB')), p)`` for every file of ``image_dir`` in sorted order, with no normalisation, resize or
mask - and its ``no_collate``.

What item ``i`` reads is decided in ``SimpleVideoReader.plan``; ``__getitem__`` reads it with Pillow and ``DeviceLoader``
(deva/inference/data/device_loader.py) decodes it on the device.
"""
import os
from os import path

import numpy as np
from PIL import Image
from torch.utils.data.dataset import Dataset

from deva.inference.data.video_reader import Plan


class SimpleVideoReader(Dataset):
    """Reads a folder of frames, one at a time: the RGB uint8 array and the file's path."""

    def __init__(self, image_dir):
        self.image_dir = image_dir
        self.frames = sorted(os.listdir(self.image_dir))

    def plan(self, idx) -> Plan:
        """What item ``idx`` reads: its frame, and nothing else."""
        return Plan(path.join(self.image_dir, self.frames[idx]), None, None, (), {})

    def __getitem__(self, idx):
        im_path = self.plan(idx).image
        return np.array(Image.open(im_path).convert('RGB')), im_path

    def __len__(self):
        return len(self.frames)


def no_collate(x):
    return x
