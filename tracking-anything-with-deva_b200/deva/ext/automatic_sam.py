"""Drop-in for the reference's deva/ext/automatic_sam.py: SAM's automatic masks -> detection id map on the device.

``segment_anything`` and the ``deva.ext.SAM`` / ``deva.ext.MobileSAM`` modules are imported by ``get_sam_model`` only,
so importing this module needs neither and does not initialise CUDA.
"""
import os
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from deva.ext.detector_masks import host_image, output_size, scored_id_map
from deva.inference.object_info import ObjectInfo


def get_sam_model(config: Dict, device: str, *, mask_generator: Optional[str] = None):
    """SAM's automatic mask generator for config['sam_variant'] ('mobile' or 'original').

    mask_generator: 'reference' (the reference's SamAutomaticMaskGenerator) or 'device' (deva.ext.sam_masks'
    DeviceMaskGenerator on the same model: the same masks, with the post-processing on the device); None reads
    DEVA_B200_SAM_MASK_GENERATOR (default 'reference')."""
    if mask_generator is None:
        mask_generator = os.environ.get('DEVA_B200_SAM_MASK_GENERATOR', 'reference')
    if mask_generator not in ('reference', 'device'):
        raise ValueError(f"mask_generator must be 'reference' or 'device', not {mask_generator!r}")
    variant = config['sam_variant'].lower()
    if variant == 'mobile':
        from deva.ext.MobileSAM.setup_mobile_sam import setup_model as setup_mobile_sam
        weights = torch.load(config['MOBILE_SAM_CHECKPOINT_PATH'])
        model = setup_mobile_sam()
        model.load_state_dict(weights, strict=True)
        model.to(device=device)
    elif variant == 'original':
        from segment_anything import sam_model_registry
        model = sam_model_registry[config['SAM_ENCODER_VERSION']](checkpoint=config['SAM_CHECKPOINT_PATH']).to(
            device=device)
    else:
        raise ValueError(f'Unknown SAM variant: {config["SAM_VARIANT"]}')
    if mask_generator == 'device':
        from deva.ext.sam_masks import DeviceMaskGenerator as Generator
    else:
        from deva.ext.SAM.automatic_mask_generator import SamAutomaticMaskGenerator as Generator
    return Generator(model,
                     points_per_side=config['SAM_NUM_POINTS_PER_SIDE'],
                     points_per_batch=config['SAM_NUM_POINTS_PER_BATCH'],
                     pred_iou_thresh=config['SAM_PRED_IOU_THRESHOLD'])


def _positive_points(config: Dict, forward_mask: torch.Tensor, device) -> np.ndarray:
    """Grid points (x, y in [0, 1]) where the blurred forward mask is background: SAM is prompted where nothing is
    tracked yet."""
    fg = F.interpolate((forward_mask > 0).float().unsqueeze(0).unsqueeze(0), scale_factor=1 / 16, mode='bilinear',
                       antialias=True)
    n = config['SAM_NUM_POINTS_PER_SIDE']
    offset = 1 / (2 * n)
    side = torch.linspace(offset, 1 - offset, n, device=device)
    points = torch.stack([side.unsqueeze(0).repeat(n, 1), side.unsqueeze(1).repeat(1, n)], dim=-1).unsqueeze(0)
    label = F.grid_sample(fg, points * 2 - 1, align_corners=False).view(-1)
    return points.view(-1, 2)[label < 0.01].cpu().numpy()


def auto_segment(config: Dict, auto_sam, image: np.ndarray, forward_mask: Optional[torch.Tensor], min_side: int,
                 suppress_small_mask: bool) -> (torch.Tensor, List[ObjectInfo]):
    """image: H*W*3 uint8 (0~255), a numpy array or a CUDA tensor; forward_mask: H*W, or None.

    Returns the int64 id map at the working resolution (shorter side ``min_side``; the image size when min_side <= 0)
    on the generator's device, and one ObjectInfo(id, score=predicted IoU) per segment.  SAM is given the host array:
    a CUDA image is downloaded once into pinned memory, a host synchronisation on top of the one the id map needs."""
    image = host_image(image)
    device = auto_sam.predictor.device
    h, w = image.shape[:2]
    new_h, new_w = output_size(h, w, min_side)
    if forward_mask is not None:
        positive_points = _positive_points(config, forward_mask, device)
        if len(positive_points) == 0:
            return torch.zeros((new_h, new_w), dtype=torch.int64, device=device), []
        mask_data = auto_sam.generate(image, positive_points, None)
    else:
        mask_data = auto_sam.generate(image)

    masks = mask_data['masks']
    if masks.shape[0] == 0:
        return torch.zeros((new_h, new_w), dtype=torch.int64, device=device), []
    id_map, segments = scored_id_map(masks.contiguous(), mask_data['iou_preds'], new_h, new_w, suppress_small_mask,
                                     config['SAM_OVERLAP_THRESHOLD'] if suppress_small_mask else 0.0)
    return id_map, [ObjectInfo(id=i, score=s) for i, s in segments]
