"""Segment Anything's automatic masks on the device, from the mask decoder's low-resolution logits.

``DeviceMaskGenerator.generate`` returns what the reference's ``SamAutomaticMaskGenerator.generate``
(deva/ext/SAM/automatic_mask_generator.py) returns for one full-frame crop: ``masks`` (bool [N, H, W] on the device),
``iou_preds``, ``points``, ``stability_score`` and ``boxes``, in the same order and with the same dtypes.  The
reference upsamples every candidate's 256x256 logits to 1024x1024 and then to the frame in float32 before it filters a
single mask; here the kernels of csrc/sam_masks.cu evaluate the same float32 values pixel by pixel and keep only
counts and boxes, so no full-resolution float mask is ever allocated, and bool masks are written for the masks that
survive the final NMS only.  Per batch of prompts there is one host synchronisation (the list of kept candidates),
plus one for the NMS result.

Crops (``crop_n_layers > 0``), ``min_mask_region_area``, ``point_grids`` and the RLE output modes are not supported:
the constructor takes only what ``deva.ext.automatic_sam.get_sam_model`` passes.  ``segment_anything`` is imported
when a generator is constructed, and CUDA is first touched by ``generate``.
"""
from typing import Dict, Optional

import numpy as np
import torch

LOW_RES = 256  # the mask decoder's logit side


def point_grid(n_per_side: int) -> np.ndarray:
    """segment_anything.utils.amg.build_point_grid: n^2 points (x, y) in [0, 1], row-major from the top left."""
    offset = 1 / (2 * n_per_side)
    side = np.linspace(offset, 1 - offset, n_per_side)
    xs = np.tile(side[None, :], (n_per_side, 1))
    ys = np.tile(side[:, None], (1, n_per_side))
    return np.stack([xs, ys], axis=-1).reshape(-1, 2)


def _upload(coords: np.ndarray, device) -> torch.Tensor:
    """torch.as_tensor(coords, device=device) without a host synchronisation: staged through pinned memory."""
    t = torch.as_tensor(coords)
    if torch.device(device).type != 'cuda':
        return t.to(device)
    return t.pin_memory().to(device, non_blocking=True)


class DeviceMaskGenerator:
    def __init__(self, model, points_per_side: int, points_per_batch: int, pred_iou_thresh: float,
                 stability_score_thresh: float = 0.95, stability_score_offset: float = 1.0,
                 box_nms_thresh: float = 0.7) -> None:
        from segment_anything.predictor import SamPredictor
        if points_per_side is None or points_per_side < 1 or points_per_batch < 1:
            raise ValueError(f'points_per_side {points_per_side} and points_per_batch {points_per_batch} must be >= 1')
        self.predictor = SamPredictor(model)
        self.point_grid = point_grid(points_per_side)
        self.points_per_batch = points_per_batch
        self.pred_iou_thresh = pred_iou_thresh
        self.stability_score_thresh = stability_score_thresh
        self.stability_score_offset = stability_score_offset
        self.box_nms_thresh = box_nms_thresh

    def _check_frame(self, h: int, w: int) -> None:
        # calculate_stability_score sums each row in int16 and the frame in int32; the kernels count in int32
        if w > 32767 or h * w >= 2 ** 31:
            raise ValueError(f'{h} x {w} frame: the stability counts overflow (width <= 32767, h * w < 2^31)')
        if h < 1 or w < 1:
            raise ValueError(f'{h} x {w} frame: empty')

    def _decode(self, points: np.ndarray, negative_points: Optional[np.ndarray], im_size):
        """The batch's prompts through the prompt encoder and mask decoder, as SamPredictor.predict_torch calls them,
        stopping at the low-resolution logits [B, 3, 256, 256] and iou_predictions [B, 3]."""
        pred = self.predictor
        if negative_points is not None:
            negative_points = np.repeat(negative_points[None, :, :], points.shape[0], axis=0)
            points = np.concatenate([points[:, None, :], negative_points], axis=1)
            in_points = _upload(pred.transform.apply_coords(points, im_size), pred.device)
            in_labels = torch.zeros((in_points.shape[0], in_points.shape[1]), dtype=torch.int, device=in_points.device)
            in_labels[:, 0] = 1
        else:
            in_points = _upload(pred.transform.apply_coords(points, im_size), pred.device)
            in_labels = torch.ones(in_points.shape[0], dtype=torch.int, device=in_points.device)
            in_points, in_labels = in_points[:, None, :], in_labels[:, None]
        model = pred.model
        sparse, dense = model.prompt_encoder(points=(in_points, in_labels), boxes=None, masks=None)
        low_res, iou = model.mask_decoder(image_embeddings=pred.features, image_pe=model.prompt_encoder.get_dense_pe(),
                                          sparse_prompt_embeddings=sparse, dense_prompt_embeddings=dense,
                                          multimask_output=True)
        return points, low_res, iou

    @torch.no_grad()
    def generate(self, image: np.ndarray, positive_points: Optional[np.ndarray] = None,
                 negative_points: Optional[np.ndarray] = None) -> Dict[str, torch.Tensor]:
        from deva import _native as nat
        h, w = image.shape[:2]
        self._check_frame(h, w)
        if positive_points is not None and len(positive_points) == 0:
            raise ValueError('positive_points is empty: the reference generator has no masks to concatenate')
        pred = self.predictor
        model = pred.model
        grid = model.image_encoder.img_size
        pred.set_image(image)
        in_h, in_w = pred.input_size
        scale = np.array((h, w))[None, ::-1]
        points_for_image = (positive_points if positive_points is not None else self.point_grid) * scale
        if negative_points is not None:
            negative_points = negative_points * scale
        thr = float(model.mask_threshold)
        thr_hi = thr + self.stability_score_offset
        thr_lo = thr - self.stability_score_offset
        use_iou = self.pred_iou_thresh > 0.0
        dev = pred.device

        kept_logits, kept_iou, kept_stab, kept_boxes, kept_points = [], [], [], [], []
        any_empty = False
        for b in range(0, len(points_for_image), self.points_per_batch):
            points, low_res, iou = self._decode(points_for_image[b:b + self.points_per_batch], negative_points,
                                                (h, w))
            logits = low_res.flatten(0, 1).float().contiguous()
            iou = iou.flatten(0, 1).float().contiguous()
            n = logits.shape[0]
            if logits.shape[1:] != (LOW_RES, LOW_RES):
                raise ValueError(f'mask decoder logits {tuple(logits.shape[1:])}, expected {LOW_RES} x {LOW_RES}')
            stats = torch.empty(n, nat.SAM_STATS, dtype=torch.int32, device=dev)
            nat.sam_mask_stats(logits, grid, in_h, in_w, h, w, iou if use_iou else None, self.pred_iou_thresh,
                               thr_hi, thr_lo, thr, stats)
            stab = torch.empty(n, dtype=torch.float32, device=dev)
            boxes = torch.empty(n, 4, dtype=torch.int64, device=dev)
            kept = torch.empty(n + 1, dtype=torch.int32, device=dev)
            nat.sam_mask_compact(stats, iou if use_iou else None, self.pred_iou_thresh, self.stability_score_thresh,
                                 stab, boxes, kept)
            kept_host = kept.cpu()  # the batch's one synchronisation
            k = int(kept_host[0])
            if k == 0:
                any_empty = True  # batched_mask_to_box gives float32 for no masks; torch.cat promotes the rest
                continue
            idx_host, idx = kept_host[1:1 + k].long(), kept[1:1 + k].long()
            kept_logits.append(logits.index_select(0, idx))
            kept_iou.append(iou.index_select(0, idx))
            kept_stab.append(stab.index_select(0, idx))
            kept_boxes.append(boxes.index_select(0, idx))
            kept_points.append(torch.as_tensor(points.repeat(3, axis=0))[idx_host])

        pred.reset_image()
        self.candidates = 0  # masks kept before the NMS, for callers that size or report the work
        point_shape = (2,) if negative_points is None else (1 + len(negative_points), 2)
        box_dtype = torch.float32 if any_empty else torch.int64
        if not kept_iou:
            return {'masks': torch.zeros(0, h, w, dtype=torch.bool, device=dev),
                    'iou_preds': torch.zeros(0, dtype=torch.float32, device=dev),
                    'points': torch.zeros((0,) + point_shape, dtype=torch.float64),
                    'stability_score': torch.zeros(0, dtype=torch.float32, device=dev),
                    'boxes': torch.zeros(0, 4, dtype=box_dtype, device=dev)}
        self.candidates = sum(t.shape[0] for t in kept_logits)
        logits = torch.cat(kept_logits)
        iou = torch.cat(kept_iou)
        stab = torch.cat(kept_stab)
        boxes = torch.cat(kept_boxes)
        points = torch.cat(kept_points)
        n = iou.numel()
        keep = torch.empty(n, dtype=torch.int64, device=dev)
        n_keep = torch.empty(1, dtype=torch.int32, device=dev)
        nat.sam_nms(boxes.float(), iou, self.box_nms_thresh, keep, n_keep)
        keep_host = torch.cat([n_keep.long(), keep]).cpu()  # the NMS result's synchronisation
        k = int(keep_host[0])
        keep, keep_host = keep[:k], keep_host[1:1 + k]
        masks = torch.empty(k, h, w, dtype=torch.bool, device=dev)
        nat.sam_mask_write(logits, keep, grid, in_h, in_w, h, w, thr, masks)
        return {'masks': masks, 'iou_preds': iou[keep], 'points': points[keep_host], 'stability_score': stab[keep],
                'boxes': boxes[keep].to(box_dtype)}
