"""Detector mask stacks -> one detection id map on the device: the pixel work of ``auto_segment`` and
``segment_with_text``.

Each composition reads the masks as bytes through the CUDA kernels (deva_b200_mask_*), brings one small per-mask table to
the host (the call's only synchronisation), applies the reference's acceptance rule there, and maps the kernel's slot
map through the resulting id table with one gather.
"""
from typing import List, Sequence, Tuple

import numpy as np
import torch

from deva import _native as nat


def output_size(h: int, w: int, min_side: int) -> Tuple[int, int]:
    """The detection map's size: the shorter side scaled to ``min_side`` (truncated), or (h, w) when min_side <= 0."""
    if min_side > 0:
        scale = min_side / min(h, w)
        return int(h * scale), int(w * scale)
    return h, w


def _to_device(array: np.ndarray, device) -> torch.Tensor:
    """Host array -> device tensor through pinned memory, without synchronising the host."""
    return torch.from_numpy(np.ascontiguousarray(array)).pin_memory().to(device, non_blocking=True)


def host_image(image):
    """A detector's input image as the host array the reference passes it.  A CUDA uint8 tensor (a frame decoded on the
    device) is downloaded into pinned memory: one host synchronisation.  Anything else is returned as it is."""
    if not (isinstance(image, torch.Tensor) and image.is_cuda and image.dtype == torch.uint8):
        return image
    host = torch.empty(image.shape, dtype=torch.uint8, pin_memory=True)
    host.copy_(image, non_blocking=True)
    torch.cuda.current_stream(image.device).synchronize()
    return host.numpy()


def _map(slot: torch.Tensor, lut: np.ndarray) -> torch.Tensor:
    return torch.index_select(_to_device(lut, slot.device), 0, slot.view(-1)).view(slot.shape)


def scored_id_map(masks: torch.Tensor, iou_preds: torch.Tensor, out_h: int, out_w: int, suppress_small_mask: bool,
                  overlap_threshold: float) -> Tuple[torch.Tensor, List[Tuple[int, float]]]:
    """auto_segment's composition.  masks bool / uint8 [n, h, w] on the device -> (int64 [out_h, out_w] id map,
    [(id, score)] of the accepted masks).

    Each pixel goes to the first maximum of [0.1, v_k * s_k] over the resized values v_k, with s = area
    (suppress_small_mask) or 2 max(area) - area.  With suppress_small_mask a mask k is accepted when it wins pixels, covers
    pixels (v > 0.5), keeps pixels (wins with v >= 0.5) and won / covered >= the threshold in float32; accepted masks
    take consecutive ids and paint the pixels they keep.  Without it the map is the winning channel itself, and the ids
    are consecutive over the masks that win a pixel."""
    device = masks.device
    n = masks.shape[0]
    if n == 0:
        return torch.zeros((out_h, out_w), dtype=torch.int64, device=device), []
    area = torch.empty(n, dtype=torch.float32, device=device)
    covered = torch.empty(n, dtype=torch.int32, device=device)
    nat.mask_stats(masks, out_h, out_w, area, covered)
    score = area if suppress_small_mask else area.max() * 2 - area
    slot = torch.empty((out_h, out_w), dtype=torch.int32, device=device)
    won = torch.empty(n + 1, dtype=torch.int32, device=device)
    kept = torch.empty(n + 1, dtype=torch.int32, device=device)
    nat.mask_scored_argmax(masks, out_h, out_w, score, suppress_small_mask, slot, won, kept)
    table = torch.stack([won[1:].double(), covered.double(), kept[1:].double(),
                         iou_preds.to(device).double()]).cpu().numpy()
    segments = []
    if not suppress_small_mask:
        for k in np.flatnonzero(table[0] > 0):
            segments.append((len(segments) + 1, float(table[3, k])))
        return slot.long(), segments
    threshold = np.float32(overlap_threshold)  # torch compares a float32 ratio with the threshold rounded to float32
    lut = np.zeros(n + 1, dtype=np.int64)
    for k in range(n):
        n_won, n_covered, n_kept = table[0, k], table[1, k], table[2, k]
        if n_won > 0 and n_covered > 0 and n_kept > 0:
            if np.float32(n_won) / np.float32(n_covered) < threshold:
                continue
            lut[k + 1] = len(segments) + 1
            segments.append((len(segments) + 1, float(table[3, k])))
    return _map(slot, lut), segments


def cover_id_map(masks: np.ndarray, out_h: int, out_w: int, device) -> Tuple[torch.Tensor, List[Tuple[int, int]]]:
    """segment_with_text's composition.  masks bool / uint8 [n, h, w] on the host -> (int64 [out_h, out_w] id map on
    ``device``, [(id, mask index)]).

    Masks are painted in descending order of source pixel count (np.flip(np.argsort) of the int64 counts), each where
    its resized value is > 0.5; a mask that covers no output pixel paints nothing and takes no id, the others take
    consecutive ids in paint order."""
    n = masks.shape[0]
    if n == 0:
        return torch.zeros((out_h, out_w), dtype=torch.int64, device=device), []
    if masks.dtype not in (np.bool_, np.uint8):
        raise TypeError(f'segment_with_text: masks are bool or uint8, not {masks.dtype}')
    areas = np.array([np.count_nonzero(m) for m in masks], dtype=np.int64)
    order = np.flip(np.argsort(areas))
    dev_masks = _to_device(np.ascontiguousarray(masks).view(np.uint8), device)
    slot = torch.empty((out_h, out_w), dtype=torch.int32, device=dev_masks.device)
    covered = torch.empty(n, dtype=torch.int32, device=dev_masks.device)
    nat.mask_last_cover(dev_masks, out_h, out_w, _to_device(order.astype(np.int32), device), slot, covered)
    covered = covered.cpu().numpy()
    lut = np.zeros(n + 1, dtype=np.int64)
    segments = []
    for i in order:
        if covered[i] > 0:
            lut[i + 1] = len(segments) + 1
            segments.append((len(segments) + 1, int(i)))
    return _map(slot, lut), segments


def stack_masks(result_masks: Sequence[np.ndarray]) -> np.ndarray:
    """np.array(result_masks), built in pinned host memory so that its upload needs no staging copy."""
    if len(result_masks) == 0:
        return np.array(result_masks)
    first = np.asarray(result_masks[0])
    if first.dtype not in (np.bool_, np.uint8):
        return np.array(result_masks)
    buf = torch.empty((len(result_masks), *first.shape), dtype=torch.bool if first.dtype == np.bool_ else torch.uint8,
                      pin_memory=True)
    out = buf.numpy()
    np.stack(result_masks, out=out)
    return out
