"""In-clip consensus when the association between detections has to be inferred
(API of the reference's deva/inference/consensus_automatic.py:82-272).

Every buffered frame's detections are projected onto a keyframe (``spatial_alignment``: one frame of the propagation
hot path, on the H100 kernels), segments of different frames that overlap with IoU > 0.5 support each other, and the
subset of segments that maximises ``sum_i x_i * (2 * support_i - 1)`` with no two overlapping segments selected is
kept.  The reference states that selection as an integer program and hands it to gurobi / pulp
(consensus_automatic.py:28-79); the constraint graph is the IoU > 0.5 match graph, so the program is a maximum-weight
independent set over small connected components and is solved here exactly, without an external solver
(``solve_exact``; ties -> the optimal selection with the lowest segment indices).  All pixel counts come from one
joint label histogram per frame pair instead of a Python loop of ``.sum().item()`` host syncs.
"""
from collections import defaultdict
from typing import Callable, Dict, List, Literal, Optional

import numpy as np
import torch

from deva.inference.consensus_associated import spatial_alignment
from deva.inference.frame_utils import FrameInfo
from deva.inference.image_feature_store import ImageFeatureStore
from deva.inference.object_info import ObjectInfo
from deva.utils.tensor_utils import pad_divide_by, unpad

_TIE = 1e-9


def solve_exact(pairwise_iou: np.ndarray, pairwise_iou_indicator: np.ndarray, total_segments: int) -> List[bool]:
    """argmax_x  sum_i x_i * (2 * sum_j iou[j, i] - 1)   s.t.  x_i + x_j <= 1 wherever indicator[i, j]
    (the program of consensus_automatic.py:28-79), solved exactly per connected component of the conflict graph."""
    weight = [float(pairwise_iou[:, i].sum() * 2) - 1.0 for i in range(total_segments)]
    nbr = [set(int(j) for j in np.nonzero(pairwise_iou_indicator[i])[0] if j != i) for i in range(total_segments)]
    selected = [False] * total_segments

    def better(a, b):  # (value, selection bitmask): higher value, then the lower bitmask
        return a[0] > b[0] + _TIE or (abs(a[0] - b[0]) <= _TIE and a[1] < b[1])

    def best_of(nodes: frozenset):
        if not nodes:
            return 0.0, 0
        v = max(nodes, key=lambda n: (len(nbr[n] & nodes), -n))
        if not (nbr[v] & nodes):  # isolated inside this sub-problem: take it iff it pays
            rest = best_of(nodes - {v})
            take = (rest[0] + weight[v], rest[1] | (1 << v))
            return take if better(take, rest) else rest
        skip = best_of(nodes - {v})
        inner = best_of(nodes - {v} - nbr[v])
        take = (inner[0] + weight[v], inner[1] | (1 << v))
        return take if better(take, skip) else skip

    seen = set()
    for s in range(total_segments):
        if s in seen:
            continue
        comp, stack = set(), [s]
        while stack:
            n = stack.pop()
            if n in comp:
                continue
            comp.add(n)
            stack.extend(nbr[n] - comp)
        seen |= comp
        _, mask = best_of(frozenset(comp))
        for n in comp:
            selected[n] = bool((mask >> n) & 1)
    return selected


def _pair_counts(mask_a: torch.Tensor, mask_b: torch.Tensor, n_labels: int) -> np.ndarray:
    """Joint label histogram of two id maps (labels < n_labels): one device reduction, one host transfer."""
    joint = mask_a.reshape(-1).long() * n_labels + mask_b.reshape(-1).long()
    return torch.bincount(joint, minlength=n_labels * n_labels).view(n_labels, n_labels).cpu().numpy()


def find_consensus_auto_association(frames: List[FrameInfo],
                                    keyframe_selection: Literal['last', 'middle', 'score', 'first'] = 'last', *,
                                    network, store: ImageFeatureStore, config: Dict,
                                    align_fn: Optional[Callable] = None) -> (int, torch.Tensor, List[ObjectInfo]):
    """Returns (keyframe time index, id mask [H,W] long on the keyframe, merged ObjectInfo list).

    ``align_fn`` (default ``spatial_alignment``) exists so tests can pin the voting logic on prescribed projections."""
    align_fn = align_fn or spatial_alignment
    time_indices = [f.ti for f in frames]
    images, masks, pads = [], [], None
    for f in frames:
        image, pads = pad_divide_by(f.image, 16)
        mask, _ = pad_divide_by(f.mask, 16)  # id map (long), not one-hot
        images.append(image)
        masks.append(mask)

    # ids that are unique across the buffered frames; one-hot float masks for the projection
    channel_to_id: List[Dict[int, int]] = []
    next_id = 0
    info_of: Dict[int, ObjectInfo] = {}
    infos_of_frame = defaultdict(list)
    for i, f in enumerate(frames):
        one_hot, mapping = [], {}
        for si, seg in enumerate(f.segments_info):
            next_id += 1
            fresh = ObjectInfo(next_id)
            fresh.copy_meta_info(seg)
            info_of[next_id] = fresh
            one_hot.append(masks[i] == seg.id)
            mapping[si] = next_id
            infos_of_frame[i].append(fresh)
        masks[i] = torch.stack(one_hot, dim=0).float() if one_hot else None
        channel_to_id.append(mapping)

    if keyframe_selection == 'last':
        keyframe_i = len(time_indices) - 1
    elif keyframe_selection == 'first':
        keyframe_i = 0
    elif keyframe_selection == 'middle':
        keyframe_i = (len(time_indices) + 1) // 2
    else:
        raise NotImplementedError
    keyframe_ti, keyframe_image, keyframe_mask = time_indices[keyframe_i], images[keyframe_i], masks[keyframe_i]

    # project every frame's segments onto the keyframe, back to id maps
    total_segments = next_id
    if total_segments == 0:
        return keyframe_ti, torch.zeros_like(frames[0].mask), []
    lut_len = 1 + max((len(m) for m in channel_to_id), default=0)
    projected: List[Optional[torch.Tensor]] = []
    for ti, image, mask, mapping in zip(time_indices, images, masks, channel_to_id):
        if mask is None:
            projected.append(None)
            continue
        if ti == keyframe_ti:
            prob = torch.cat([torch.ones_like(keyframe_mask[0:1]) * 0.5, keyframe_mask], dim=0)
        else:
            prob = align_fn(ti, image, mask, keyframe_ti, keyframe_image, network, store, config)[0]
        channel = torch.argmax(unpad(prob, pads), dim=0)
        lut = torch.zeros(lut_len, dtype=torch.long, device=channel.device)
        for channel_id, object_id in mapping.items():
            lut[channel_id + 1] = object_id  # +1: channel 0 is the background
        projected.append(lut[channel])

    n_labels = total_segments + 1
    area = np.zeros(n_labels, dtype=np.int64)
    for pm in projected:
        if pm is not None:
            area += torch.bincount(pm.reshape(-1), minlength=n_labels).cpu().numpy()

    # pairwise IoU between segments of different frames (upper triangle: ids grow with the frame index)
    matching_table = defaultdict(list)
    pairwise_iou = np.zeros((total_segments, total_segments), dtype=np.float32)
    for i in range(len(frames)):
        if projected[i] is None:
            continue
        for j in range(i + 1, len(frames)):
            if projected[j] is None:
                continue
            counts = _pair_counts(projected[i], projected[j], n_labels)
            for isthing_status in (None, False, True):
                taken = set()
                for obj1 in infos_of_frame[i]:
                    if obj1.isthing != isthing_status:
                        continue
                    for obj2 in infos_of_frame[j]:
                        if obj2.isthing != isthing_status or obj2.id in taken:
                            continue
                        inter = int(counts[obj1.id, obj2.id])
                        if inter == 0:
                            continue
                        iou = inter / (int(area[obj1.id]) + int(area[obj2.id]) - inter)
                        if iou > 0.5:  # unique per segment, so the first hit is the only one
                            matching_table[obj1.id].append(obj2.id)
                            matching_table[obj2.id].append(obj1.id)
                            taken.add(obj2.id)
                            pairwise_iou[obj1.id - 1, obj2.id - 1] = iou
                            break

    pairwise_iou = pairwise_iou + pairwise_iou.T
    indicator = pairwise_iou > 0.49
    pairwise_iou = pairwise_iou * indicator
    results = solve_exact(pairwise_iou, indicator, total_segments)

    output_mask = torch.zeros_like(frames[0].mask)
    output_info, chosen_area = [], {}
    for channel_id, selected in enumerate(results):
        if selected:
            object_id = channel_id + 1
            chosen_area[object_id] = int(area[object_id])
            merged = info_of[object_id]
            for other in matching_table[object_id]:
                merged.merge(info_of[other])
            output_info.append(merged)
    if chosen_area:  # paint large segments first so that small ones stay visible
        for object_id, _ in sorted(chosen_area.items(), key=lambda kv: kv[1], reverse=True):
            frame_i = next(i for i, m in enumerate(channel_to_id) if object_id in m.values())
            output_mask[projected[frame_i] == object_id] = object_id
    return keyframe_ti, output_mask, output_info
