"""Oracle of deva/ext/sam_masks.py: the device mask generator's algorithm restated on the CPU with torch.

Per batch of prompts: the low-resolution logits and predicted IoUs from the model's prompt encoder and mask decoder;
the predicted-IoU filter; for the candidates that pass it, Sam.postprocess_masks' two bilinear stages with torch's CPU
``F.interpolate`` (the crop in between), the three counts of calculate_stability_score and the box of the pixels above
the mask threshold; stability = intersections / unions and its filter.  Then torchvision's CPU ``batched_nms`` with one
category, and the kept masks thresholded.  The output is the reference generator's MaskData fields.

``reference_generator()`` loads the reference's SamAutomaticMaskGenerator (staged unmodified under
``oracle/_ref/deva/ext/SAM`` by build_ref_sam.py) by path, over the stand-in ``segment_anything`` of sam_stub.py.
"""
import importlib.util
import os
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle import sam_stub

HERE = os.path.dirname(os.path.abspath(__file__))
REF_GENERATOR = os.path.join(HERE, '_ref', 'deva', 'ext', 'SAM', 'automatic_mask_generator.py')


def reference_available() -> bool:
    return os.path.isfile(REF_GENERATOR)


def reference_generator():
    """The reference's SamAutomaticMaskGenerator class; installs the stand-in segment_anything."""
    sam_stub.install()
    spec = importlib.util.spec_from_file_location('ref_sam_automatic_mask_generator', REF_GENERATOR)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.SamAutomaticMaskGenerator


def upsample(logits: torch.Tensor, grid: int, input_size, original_size) -> torch.Tensor:
    """Sam.postprocess_masks of [n, lh, lw] logits -> [n, H, W] float32."""
    m = F.interpolate(logits[:, None], (grid, grid), mode='bilinear', align_corners=False)
    m = m[..., :input_size[0], :input_size[1]]
    return F.interpolate(m, tuple(original_size), mode='bilinear', align_corners=False)[:, 0]


def mask_stats(logits, grid, input_size, original_size, thr_hi, thr_lo, thr, chunk=16):
    """-> int64 [n, 7]: pixels > thr_hi, > thr_lo, > thr, then x0, y0, x1, y1 of the pixels > thr (0s when none)."""
    out = torch.zeros(logits.shape[0], 7, dtype=torch.int64)
    for s in range(0, logits.shape[0], chunk):
        v = upsample(logits[s:s + chunk], grid, input_size, original_size)
        m = v > thr
        out[s:s + chunk, 0] = (v > thr_hi).flatten(1).sum(1)
        out[s:s + chunk, 1] = (v > thr_lo).flatten(1).sum(1)
        out[s:s + chunk, 2] = m.flatten(1).sum(1)
        rows, cols = m.any(2), m.any(1)
        for j in range(m.shape[0]):
            if out[s + j, 2] > 0:
                ys, xs = torch.nonzero(rows[j])[:, 0], torch.nonzero(cols[j])[:, 0]
                out[s + j, 3:] = torch.stack([xs.min(), ys.min(), xs.max(), ys.max()])
    return out


@torch.no_grad()
def generate(model, image: np.ndarray, points_per_side: int, points_per_batch: int, pred_iou_thresh: float,
             stability_score_thresh: float = 0.95, stability_score_offset: float = 1.0, box_nms_thresh: float = 0.7,
             positive_points: Optional[np.ndarray] = None,
             negative_points: Optional[np.ndarray] = None) -> Dict[str, torch.Tensor]:
    from torchvision.ops.boxes import batched_nms
    h, w = image.shape[:2]
    if positive_points is not None and len(positive_points) == 0:
        raise ValueError('positive_points is empty')
    pred = sam_stub.SamPredictor(model)
    pred.set_image(image)
    grid = model.image_encoder.img_size
    thr = float(model.mask_threshold)
    scale = np.array((h, w))[None, ::-1]
    pts_all = (positive_points if positive_points is not None else sam_stub.build_point_grid(points_per_side)) * scale
    neg = None if negative_points is None else negative_points * scale
    logits_k, iou_k, stab_k, box_k, pts_k = [], [], [], [], []
    any_empty = False
    for b in range(0, len(pts_all), points_per_batch):
        points = pts_all[b:b + points_per_batch]
        if neg is not None:
            points = np.concatenate([points[:, None, :], np.repeat(neg[None], points.shape[0], axis=0)], axis=1)
            labels = torch.zeros(points.shape[:2], dtype=torch.int)
            labels[:, 0] = 1
            coords = torch.as_tensor(pred.transform.apply_coords(points, (h, w)))
        else:
            coords = torch.as_tensor(pred.transform.apply_coords(points, (h, w)))[:, None, :]
            labels = torch.ones(coords.shape[0], 1, dtype=torch.int)
        sparse, dense = model.prompt_encoder(points=(coords, labels), boxes=None, masks=None)
        low_res, iou = model.mask_decoder(image_embeddings=pred.features, image_pe=model.prompt_encoder.get_dense_pe(),
                                          sparse_prompt_embeddings=sparse, dense_prompt_embeddings=dense,
                                          multimask_output=True)
        low_res, iou = low_res.flatten(0, 1), iou.flatten(0, 1)
        cand = torch.nonzero(iou > pred_iou_thresh)[:, 0] if pred_iou_thresh > 0.0 else torch.arange(iou.numel())
        st = mask_stats(low_res[cand], grid, pred.input_size, (h, w), thr + stability_score_offset,
                        thr - stability_score_offset, thr)
        stab = st[:, 0].to(torch.int32) / st[:, 1].to(torch.int32)
        ok = stab >= stability_score_thresh if stability_score_thresh > 0.0 else torch.ones_like(stab, dtype=torch.bool)
        sel = cand[ok]
        if sel.numel() == 0:
            any_empty = True
            continue
        logits_k.append(low_res[sel])
        iou_k.append(iou[sel])
        stab_k.append(stab[ok])
        box_k.append(st[ok, 3:])
        pts_k.append(torch.as_tensor(points.repeat(3, axis=0))[sel])
    box_dtype = torch.float32 if any_empty else torch.int64
    if not iou_k:
        shape = (2,) if neg is None else (1 + len(neg), 2)
        return {'masks': torch.zeros(0, h, w, dtype=torch.bool), 'iou_preds': torch.zeros(0),
                'points': torch.zeros((0,) + shape, dtype=torch.float64), 'stability_score': torch.zeros(0),
                'boxes': torch.zeros(0, 4, dtype=box_dtype)}
    logits, iou, stab = torch.cat(logits_k), torch.cat(iou_k), torch.cat(stab_k)
    boxes, points = torch.cat(box_k), torch.cat(pts_k)
    keep = batched_nms(boxes.float(), iou, torch.zeros_like(boxes[:, 0]), iou_threshold=box_nms_thresh)
    masks = torch.cat([upsample(logits[keep[s:s + 16]], grid, pred.input_size, (h, w)) > thr
                       for s in range(0, keep.numel(), 16)]) if keep.numel() else torch.zeros(0, h, w, dtype=torch.bool)
    return {'masks': masks, 'iou_preds': iou[keep], 'points': points[keep], 'stability_score': stab[keep],
            'boxes': boxes[keep].to(box_dtype)}
