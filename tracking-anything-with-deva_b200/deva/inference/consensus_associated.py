"""In-clip consensus when the association between detections is already known
(API of the reference's deva/inference/consensus_associated.py:16-147).

``spatial_alignment`` is one frame of exactly the propagation hot path - encode the source mask into values,
read them from the target frame's query, decode - so it runs on the same kernels as ``DEVAInferenceCore.step``:
the source frame becomes a one-frame bank of a throw-away ``MemoryManager`` (token-major fp16 values, split-fp16 keys)
and the read is the fused similarity/top-k/softmax/readout path.
"""
from typing import Dict, List, Optional

import torch

from deva.inference.image_feature_store import ImageFeatureStore
from deva.inference.memory_manager import MemoryManager
from deva.utils.tensor_utils import pad_divide_by, unpad


def spatial_alignment(src_ti: int, src_image: torch.Tensor, src_mask: torch.Tensor, tar_ti: int,
                      tar_image: torch.Tensor, network, store: ImageFeatureStore, config: Dict) -> torch.Tensor:
    """Project ``src_mask`` [K,H,W] (float, one channel per object) of the source frame onto the target frame.

    Returns the target-frame probabilities [1, K+1, H, W] (channel 0 = background), like
    consensus_associated.py:16-69: values of the source masks are read with the target's query
    (``get_similarity`` -> ``do_softmax(top_k)`` -> ``value @ affinity``) and decoded with a zero-initialised,
    deep-updated sensory state and the source mask as ``last_mask``.
    """
    num_objects, h, w = src_mask.shape
    src_image = src_image.unsqueeze(0)
    tar_image = tar_image.unsqueeze(0)
    src_mask = src_mask.unsqueeze(0)

    src_ms_features = store.get_ms_features(src_ti, src_image)
    src_key, src_shrinkage, src_selection = store.get_key(src_ti, src_image)
    tar_ms_features = store.get_ms_features(tar_ti, tar_image)
    tar_key, _, tar_selection = store.get_key(tar_ti, tar_image)

    sensory = torch.zeros((1, num_objects, config['value_dim'], h // 16, w // 16), device=src_key.device)
    value, sensory = network.encode_mask(src_image, src_ms_features, sensory, src_mask, is_deep_update=True,
                                         chunk_size=config['chunk_size'])

    # the source frame as a one-frame memory bank (no long-term logic: nothing is consolidated or counted)
    bank = MemoryManager(dict(config, enable_long_term=False, enable_long_term_count_usage=False))
    bank.work_frames_without_long_term = 1
    objects = list(range(1, num_objects + 1))
    bank.add_memory(src_key, src_shrinkage, value, objects, selection=src_selection)
    readout = bank.match_memory(tar_key, tar_selection)
    parts = [readout[o] for o in objects]
    first = parts[0]
    if num_objects > 1 and all(p.untyped_storage().data_ptr() == first.untyped_storage().data_ptr() and
                               p.stride() == first.stride() for p in parts):  # consecutive slices of one buffer
        step = parts[1].storage_offset() - first.storage_offset()
        memory_readout = first.as_strided((num_objects, *first.shape), (step, *first.stride()), first.storage_offset())
    else:
        memory_readout = torch.stack(parts, dim=0)
    memory_readout = memory_readout.unsqueeze(0)

    _, _, tar_mask = network.segment(tar_ms_features, memory_readout, sensory, src_mask,
                                     chunk_size=config['chunk_size'], update_sensory=False)
    return tar_mask


def _keyframe_objective_from_mask(mask: torch.Tensor, score: Optional[float], method: str = 'high_foreground') -> float:
    """How good a keyframe would this detection make (consensus_associated.py:72-79)."""
    if method == 'high_foreground':
        return float((mask > 0.8).float().mean())
    if method == 'score':
        return score
    raise NotImplementedError


def find_consensus_with_established_association(time_indices: List[int], images: List[torch.Tensor],
                                                masks: List[torch.Tensor], network, store: ImageFeatureStore,
                                                config: Dict, scores: List[float] = None) -> (int, torch.Tensor):
    """Weighted average, on the best keyframe, of every frame's masks projected onto it
    (consensus_associated.py:82-147).  ``images`` / ``masks`` are padded in place like the reference does.
    Returns (keyframe time index, soft masks [K, H, W] cropped to the un-padded size)."""
    pads = None
    for i, (image, mask) in enumerate(zip(images, masks)):
        images[i], pads = pad_divide_by(image, 16)
        masks[i], _ = pad_divide_by(mask, 16)

    use_score = scores is not None
    if scores is None:
        scores = [1 for _ in time_indices]
    scores = torch.softmax(torch.Tensor(scores) * 2, dim=0).tolist()

    best = float('-inf')
    keyframe_ti = keyframe_image = keyframe_mask = keyframe_score = None
    for ti, image, mask, score in zip(time_indices, images, masks, scores):
        objective = _keyframe_objective_from_mask(mask, score, method='score' if use_score else 'high_foreground')
        if objective > best:
            best = objective
            keyframe_ti, keyframe_image, keyframe_mask = ti, image, mask
            keyframe_score = score if use_score else None
    if keyframe_score is None:
        keyframe_score = scores[0]

    total = keyframe_mask * keyframe_score
    for ti, image, mask, score in zip(time_indices, images, masks, scores):
        if ti == keyframe_ti:
            continue
        projected = spatial_alignment(ti, image, mask, keyframe_ti, keyframe_image, network, store, config)
        total = total + projected[0, 1:] * score
    return keyframe_ti, unpad(total, pads)
