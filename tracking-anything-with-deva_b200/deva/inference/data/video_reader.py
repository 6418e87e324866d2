"""``VideoReader``: one video's frames and masks, item for item what the reference's reader gives (same constructor,
attributes and Pillow / torchvision calls).

What item ``i`` reads is decided in one place, ``VideoReader.plan``: the frame, where its shape comes from, which mask
files are read and how, and the info fields.  ``__getitem__`` runs the plan with Pillow and torchvision; ``DeviceLoader``
(deva/inference/data/device_loader.py) runs the same plan on the device.  pycocotools is imported only when masks come
from ``segmentation_from_dict``, so the reader imports without it.
"""
import copy
import os
from os import path
from typing import Dict, List, NamedTuple, Optional, Tuple

import numpy as np
import torch
from PIL import Image
from torch.utils.data.dataset import Dataset
from torchvision import transforms
from torchvision.transforms import InterpolationMode

from deva.inference.frame_io import IMAGENET_MEAN, IMAGENET_STD

im_normalization = transforms.Normalize(mean=list(IMAGENET_MEAN), std=list(IMAGENET_STD))

# how a plan's mask files are read
MASK_ID = 'id'                  # one optional index PNG, convert('P'), Resize(NEAREST) -> int64 and its labels
MASK_SOFT = 'soft'              # one L PNG (a single object, or object_name's folder), Resize(BILINEAR) / 255
MASK_SOFT_MULTI = 'soft_multi'  # one L PNG per prob folder, each asserted to exist, stacked
MASK_DETECTION = 'detection'    # one optional P / L / RGB PNG -> int32 ids (DetectionVideoReader)
MASK_DICT = 'dict'              # a COCO RLE from segmentation_from_dict


class Plan(NamedTuple):
    """What item ``i`` of a reader reads.  ``info`` holds the item's info fields in the reader's order, with
    ``shape`` (and ``is_rgb`` for detections) still None; ``masks`` the mask paths for ``mask_kind`` (None: no mask)."""
    image: str
    size_path: Optional[str]  # None: the shape is the frame's own
    mask_kind: Optional[str]
    masks: Tuple[str, ...]
    info: Dict


def reader_transforms(size: int, soft: bool):
    """(im_transform, mask_transform) of the readers at ``size`` (< 0: no resize)."""
    if size < 0:
        return transforms.Compose([transforms.ToTensor(), im_normalization]), transforms.Compose([])
    im = transforms.Compose([transforms.ToTensor(), im_normalization,
                             transforms.Resize(size, interpolation=InterpolationMode.BILINEAR, antialias=True)])
    mode = InterpolationMode.BILINEAR if soft else InterpolationMode.NEAREST
    mask = transforms.Compose([transforms.Resize(size, interpolation=mode, antialias=True) if soft else
                               transforms.Resize(size, interpolation=mode)])
    return im, mask


def read_frame(reader, plan: Plan):
    """The plan's frame through ``reader.im_transform`` and its shape (h, w), read with Pillow."""
    img = Image.open(plan.image).convert('RGB')
    if plan.size_path is None:
        shape = np.array(img).shape[:2]
    else:
        shape = np.array(Image.open(plan.size_path).convert('RGB')).shape[:2]
    return reader.im_transform(img), shape


class VideoReader(Dataset):
    """Reads one video, one frame at a time.

    image_dir: the video's frames; mask_dir: its PNG masks.  size: resize the short side to ``size`` (< 0: keep).
    to_save: frame names (without extension) whose results are saved (None: all).  use_all_masks: read every mask
    in mask_dir, not only the first.  size_dir: frames whose shape is reported (default image_dir).  start / end /
    num_sampled_frames / reverse / enabled_frame_list select frames.  soft_mask: read probability masks from
    sub-folders (all, or ``object_name``'s; ``multi_object=False``: mask_dir itself).  segmentation_from_dict: read
    masks as COCO RLE from this dict instead."""

    def __init__(self, vid_name, image_dir, mask_dir, *, size=-1, to_save=None, use_all_masks=False, size_dir=None,
                 start=-1, end=-1, num_sampled_frames=-1, reverse=False, soft_mask=False, object_name=None,
                 multi_object=True, segmentation_from_dict: Optional[Dict[str, Dict]] = None,
                 enabled_frame_list: Optional[List[str]] = None):
        self.vid_name = vid_name
        self.image_dir = image_dir
        self.mask_dir = mask_dir
        self.to_save = to_save
        self.use_all_mask = use_all_masks
        self.soft_mask = soft_mask
        self.object_name = object_name
        self.multi_object = multi_object
        self.segmentation_from_dict = segmentation_from_dict
        self.enabled_frame_list = enabled_frame_list
        self.size_dir = self.image_dir if size_dir is None else size_dir

        listed = sorted(os.listdir(self.image_dir))
        if segmentation_from_dict is None:
            frames = listed
        else:  # the dict's keys, with the image directory's extension
            frames = [key + listed[0][-4:] for key in sorted(segmentation_from_dict.keys())]
        if enabled_frame_list is not None:
            frames = [f for f in frames if f[:-4] in enabled_frame_list]
        self.frames = frames
        self._all_frames = copy.deepcopy(frames)
        if start >= 0:
            frames = frames[start:end] if end >= 0 else frames[start:]
        elif end >= 0:
            frames = frames[:end]
        if num_sampled_frames > 0:  # m evenly spaced frames, each in the middle of its share
            assert start < 0 and end < 0
            n = len(frames)
            m = min(num_sampled_frames, n)
            frames = [frames[k * n // m + n // (2 * m)] for k in range(m)]
        if reverse:
            frames = list(reversed(frames))
        self.frames = frames

        if segmentation_from_dict is not None:
            self.palette = None
            self.first_mask_frame = self.frames[0]
        elif soft_mask:
            self.palette = None
            if multi_object and object_name is not None:
                self.mask_dir = path.join(self.mask_dir, object_name)
                self.first_mask_frame = sorted(os.listdir(self.mask_dir))[0]
            elif multi_object:
                self.prob_folders = [f for f in sorted(os.listdir(self.mask_dir)) if '.csv' not in f]
                self.first_mask_frame = sorted(os.listdir(path.join(self.mask_dir, self.prob_folders[0])))[0]
            else:
                self.mask_dir = path.join(self.mask_dir)
                self.first_mask_frame = sorted(os.listdir(self.mask_dir))[0]
        else:
            self.palette = Image.open(path.join(mask_dir, sorted(os.listdir(mask_dir))[0])).getpalette()
            self.first_mask_frame = sorted(os.listdir(self.mask_dir))[0]

        self.im_transform, self.mask_transform = reader_transforms(size, soft_mask)
        self.size = size

    def plan(self, idx) -> Plan:
        """What item ``idx`` reads (see ``Plan``)."""
        frame = self.frames[idx]
        stem = frame[:-4]
        info = {'frame': frame, 'save': (self.to_save is None) or (stem in self.to_save)}
        kind, masks = None, ()
        if self.use_all_mask or stem == self.first_mask_frame[:-4]:
            if self.segmentation_from_dict is not None:
                kind = MASK_DICT
            elif self.soft_mask and (self.object_name is not None or not self.multi_object):
                kind, masks = MASK_SOFT, (path.join(self.mask_dir, stem + '.png'),)
                if self.object_name is not None:
                    info['object_name'] = self.object_name
            elif self.soft_mask:
                kind = MASK_SOFT_MULTI
                masks = tuple(path.join(self.mask_dir, folder, stem + '.png') for folder in self.prob_folders)
            else:
                kind, masks = MASK_ID, (path.join(self.mask_dir, stem + '.png'),)
        im_path = path.join(self.image_dir, frame)
        info.update(shape=None, need_resize=not (self.size < 0), time_index=self._all_frames.index(frame),
                    path_to_image=im_path)
        return Plan(im_path, None if self.image_dir == self.size_dir else path.join(self.size_dir, frame), kind, masks,
                    info)

    def assemble(self, plan: Plan, rgb, shape, mask=None, valid_labels=None):
        """The item of ``plan`` from its frame, shape and (optional) mask and labels."""
        data = {}
        if mask is not None:
            data['mask'] = mask
            data['valid_labels'] = valid_labels
        info = dict(plan.info)
        info['shape'] = shape
        data['rgb'] = rgb
        data['info'] = info
        return data

    def read_masks(self, plan: Plan):
        """(mask, valid_labels) of the plan, read with Pillow; (None, None) without one."""
        if plan.mask_kind == MASK_DICT:
            import pycocotools.mask as mask_utils
            pred = self.segmentation_from_dict[plan.info['frame'][:-4]][self.object_name]
            mask = self.mask_transform(mask_utils.decode(pred['segmentation']))
            return torch.FloatTensor(np.array(mask)).unsqueeze(0), torch.LongTensor([1])
        if plan.mask_kind in (MASK_SOFT, MASK_SOFT_MULTI):
            planes = []
            for mask_path in plan.masks:
                if plan.mask_kind == MASK_SOFT_MULTI:
                    assert path.exists(mask_path)
                planes.append(torch.FloatTensor(np.array(self.mask_transform(Image.open(mask_path)))) / 255)
            planes = torch.stack(planes, dim=0)
            return planes, torch.LongTensor(list(range(1, len(planes) + 1)))
        if plan.mask_kind == MASK_ID and path.exists(plan.masks[0]):
            mask = torch.LongTensor(np.array(self.mask_transform(Image.open(plan.masks[0]).convert('P'))))
            labels = torch.unique(mask)
            return mask, labels[labels != 0]
        return None, None

    def __getitem__(self, idx):
        plan = self.plan(idx)
        rgb, shape = read_frame(self, plan)
        mask, labels = self.read_masks(plan)
        return self.assemble(plan, rgb, shape, mask, labels)

    def get_palette(self):
        return self.palette

    def __len__(self):
        return len(self.frames)
