"""``DetectionVideoReader``: one video's frames and per-frame detection masks, item for item what the reference's
reader gives.  Its plan (``DetectionVideoReader.plan``) is run by ``__getitem__`` with Pillow and by ``DeviceLoader``
on the device.

The reference's quirks are kept: ``is_rgb`` carries over from the last mask read (None before the first, which
``default_collate`` rejects), and ``reverse=True`` makes ``frames`` an iterator, so the constructor fails."""
import os
from os import path

import numpy as np
from PIL import Image
from torch.utils.data.dataset import Dataset

from deva.inference.data.video_reader import MASK_DETECTION, Plan, read_frame, reader_transforms


class DetectionVideoReader(Dataset):
    """Reads one video, one frame at a time, with the detection mask (P / L index or RGB id PNG) and the JSON of each
    frame when mask_dir has them.  size: resize the short side to ``size`` (< 0: keep).  to_save: frame names
    (without extension) whose results are saved (None: all).  size_dir: frames whose shape is reported."""

    def __init__(self, vid_name, image_dir, mask_dir, size=-1, to_save=None, size_dir=None, start=-1, end=-1,
                 reverse=False):
        self.vid_name = vid_name
        self.image_dir = image_dir
        self.mask_dir = mask_dir
        self.to_save = to_save
        self.size_dir = self.image_dir if size_dir is None else size_dir

        self.frames = sorted(os.listdir(self.image_dir))
        if start > 0:
            self.frames = self.frames[start:]
        if end > 0:
            self.frames = self.frames[:end]
        if reverse:
            self.frames = reversed(self.frames)

        first_png = self.frames[0].replace('.jpg', '.png')
        self.palette = Image.open(path.join(mask_dir, first_png)).getpalette()
        self.first_gt_path = path.join(self.mask_dir, first_png)

        self.im_transform, self.mask_transform = reader_transforms(size, False)
        self.size = size
        self.is_rgb = None

    def plan(self, idx) -> Plan:
        """What item ``idx`` reads (see ``video_reader.Plan``); the mask is read when its file exists."""
        frame = self.frames[idx]
        stem = frame[:-4]
        info = {'frame': frame, 'save': (self.to_save is None) or (stem in self.to_save)}
        json_path = path.join(self.mask_dir, stem + '.json')
        if path.exists(json_path):
            info['json'] = json_path
        im_path = path.join(self.image_dir, frame)
        info.update(is_rgb=None, shape=None, need_resize=not (self.size < 0), path_to_image=im_path)
        return Plan(im_path, None if self.image_dir == self.size_dir else path.join(self.size_dir, frame),
                    MASK_DETECTION, (path.join(self.mask_dir, stem + '.png'),), info)

    def assemble(self, plan: Plan, rgb, shape, mask=None, is_rgb=None):
        """The item of ``plan`` from its frame, shape and (optional) id mask; reading a mask sets ``self.is_rgb``."""
        data = {}
        if mask is not None:
            self.is_rgb = is_rgb
            data['mask'] = mask
        info = dict(plan.info)
        info['is_rgb'] = self.is_rgb
        info['shape'] = shape
        data['rgb'] = rgb
        data['info'] = info
        return data

    def read_mask(self, plan: Plan):
        """(int32 id mask, is_rgb) of the plan, read with Pillow; (None, None) when the file does not exist."""
        if not path.exists(plan.masks[0]):
            return None, None
        mask = self.mask_transform(Image.open(plan.masks[0]))
        if mask.mode == 'RGB':
            mask = np.array(mask, dtype=np.int32)
            return mask[:, :, 0] + mask[:, :, 1] * 256 + mask[:, :, 2] * 256 * 256, True
        return np.array(mask.convert('P'), dtype=np.int32), False

    def __getitem__(self, idx):
        plan = self.plan(idx)
        rgb, shape = read_frame(self, plan)
        mask, is_rgb = self.read_mask(plan)
        return self.assemble(plan, rgb, shape, mask, is_rgb)

    def get_palette(self):
        return self.palette

    def __len__(self):
        return len(self.frames)
