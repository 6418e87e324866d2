"""Per-frame propagation state machine (API of deva/inference/inference_core.py:17-290).

``DEVAInferenceCore`` keeps the reference's constructor, methods, attributes and side effects so that
``evaluation/eval_vos.py`` and the ``deva/ext`` detector hooks can drive it unchanged; the work it
schedules runs on the H100 kernels (memory read / bank) and the engine (conv stack).
"""
import warnings
from typing import Dict, Iterable, List, Literal, Optional

import torch

from deva.inference.consensus_automatic import find_consensus_auto_association
from deva.inference.frame_utils import FrameInfo
from deva.inference.image_feature_store import ImageFeatureStore
from deva.inference.memory_manager import MemoryManager
from deva.inference.object_info import ObjectInfo
from deva.inference.object_manager import ObjectManager
from deva.inference.segment_merging import match_and_merge
from deva.utils.tensor_utils import pad_divide_by, unpad


class DEVAInferenceCore:
    def __init__(self, network, config: Dict, *, image_feature_store: ImageFeatureStore = None):
        self.network = network
        self.config = config
        self.mem_every = config['mem_every']
        self.enable_long_term = config['enable_long_term']
        self.chunk_size = config['chunk_size']
        self.max_missed_detection_count = config.get('max_missed_detection_count')
        self.max_num_objects = config.get('max_num_objects')

        self.curr_ti = -1
        self.last_mem_ti = 0
        self.memory = MemoryManager(config=config)
        self.object_manager = ObjectManager()
        self.image_feature_store = image_feature_store or ImageFeatureStore(self.network)
        self.last_mask = None
        self.pad = None
        self.frame_buffer: List[FrameInfo] = []  # semi-online processing

    # ------------------------------------------------------------------ id mode
    def enabled_long_id(self) -> None:
        self.object_manager.use_long_id = True

    @property
    def use_long_id(self):
        return self.object_manager.use_long_id

    # ------------------------------------------------------------------ building blocks
    def _features(self, image_ti: int, image: torch.Tensor):
        ms = self.image_feature_store.get_ms_features(image_ti, image)
        return (ms, *self.image_feature_store.get_key(image_ti, image))

    def _add_memory(self, image: torch.Tensor, ms_features: Iterable[torch.Tensor], prob: torch.Tensor,
                    key: torch.Tensor, shrinkage: torch.Tensor, selection: torch.Tensor, *,
                    is_deep_update: bool = True) -> None:
        """image [1,3,H,W]; prob [1,K,H,W] in [0,1]  (inference_core.py:55-87)."""
        if prob.shape[1] == 0:
            warnings.warn('Empty object mask!', RuntimeWarning)
            return
        ids = self.object_manager.all_obj_ids
        self.memory.initialize_sensory_if_needed(key, ids)
        value, sensory = self.network.encode_mask(image, ms_features, self.memory.get_sensory(ids), prob,
                                                  is_deep_update=is_deep_update, chunk_size=self.chunk_size)
        self.memory.add_memory(key, shrinkage, value, ids, selection=selection)
        self.last_mem_ti = self.curr_ti
        if is_deep_update:
            self.memory.update_sensory(sensory, ids)

    def _segment(self, key: torch.Tensor, selection: torch.Tensor, ms_features: Iterable[torch.Tensor],
                 update_sensory: bool = True) -> torch.Tensor:
        """Memory read + decode -> prob [K+1,H,W]  (inference_core.py:89-113)."""
        if not self.memory.engaged:
            warnings.warn('Trying to segment without any memory!', RuntimeWarning)
            return torch.zeros((1, key.shape[-2] * 16, key.shape[-1] * 16), device=key.device, dtype=key.dtype)
        ids = self.object_manager.all_obj_ids
        readout = self.object_manager.realize_dict(self.memory.match_memory(key, selection)).unsqueeze(0)
        sensory, _, prob = self.network.segment(ms_features, readout, self.memory.get_sensory(ids), self.last_mask,
                                                chunk_size=self.chunk_size, update_sensory=update_sensory)
        if update_sensory:
            self.memory.update_sensory(sensory, ids)
        return prob[0]

    # ------------------------------------------------------------------ semi-online buffer
    def add_to_temporary_buffer(self, frame_info: FrameInfo) -> None:
        self.frame_buffer.append(frame_info)

    def vote_in_temporary_buffer(self, keyframe_selection: Literal['last', 'middle', 'score', 'first'] = 'first'
                                 ) -> (int, torch.Tensor, List[ObjectInfo]):
        """In-clip consensus over the buffered detections (inference_core.py:118-130)."""
        return find_consensus_auto_association(self.frame_buffer, network=self.network,
                                               store=self.image_feature_store, config=self.config,
                                               keyframe_selection=keyframe_selection)

    def clear_buffer(self) -> None:
        for f in self.frame_buffer:
            self.image_feature_store.delete(f.ti)
        self.frame_buffer = []

    # ------------------------------------------------------------------ detections
    def incorporate_detection(self, image: torch.Tensor, new_mask: torch.Tensor, segments_info: List[ObjectInfo], *,
                              image_ti_override: bool = None, forward_mask: torch.Tensor = None,
                              incremental: bool = False) -> torch.Tensor:
        """Merge an image-level detection into the propagated state (inference_core.py:137-198)."""
        self.curr_ti += 1
        image_ti = self.curr_ti if image_ti_override is None else image_ti_override
        image, self.pad = pad_divide_by(image, 16)
        new_mask, _ = pad_divide_by(new_mask, 16)
        image = image.unsqueeze(0)
        ms_features, key, shrinkage, selection = self._features(image_ti, image)

        if forward_mask is None:
            if self.memory.engaged:
                forward_mask = torch.argmax(self._segment(key, selection, ms_features), dim=0)
            else:
                forward_mask = torch.zeros_like(new_mask)

        merged = match_and_merge(forward_mask, new_mask, self.object_manager, segments_info,
                                 max_num_objects=self.max_num_objects, incremental_mode=incremental)
        purged, tmp_keep, obj_keep = self.object_manager.purge_inactive_objects(self.max_missed_detection_count)
        if purged:
            self.memory.purge_except(obj_keep)
            merged = merged[[t - 1 for t in tmp_keep]]

        self.last_mask = merged.unsqueeze(0).type_as(key)
        self._add_memory(image, ms_features, self.last_mask, key, shrinkage, selection)
        prob = self.network.aggregate(self.last_mask[0], dim=0)
        self.image_feature_store.delete(image_ti)
        return unpad(prob, self.pad)

    # ------------------------------------------------------------------ the per-frame step
    def step(self, image: torch.Tensor, mask: torch.Tensor = None, objects: Optional[List[int]] = None, *,
             hard_mask: bool = True, end: bool = False, image_ti_override: bool = None,
             delete_buffer: bool = True) -> torch.Tensor:
        """image [3,H,W]; mask [H,W] ids (hard) or [K,H,W] probabilities (soft) or None.

        Returns prob [(K+1),H,W], channel 0 = background, channel i = temporary id i
        (inference_core.py:200-290).
        """
        if objects is None and mask is not None:
            assert not hard_mask
            objects = list(range(1, mask.shape[0] + 1))
        self.curr_ti += 1
        image_ti = self.curr_ti if image_ti_override is None else image_ti_override
        image, self.pad = pad_divide_by(image, 16)
        image = image.unsqueeze(0)

        is_mem_frame = ((self.curr_ti - self.last_mem_ti >= self.mem_every) or (mask is not None)) and not end
        need_segment = (mask is None) or (self.object_manager.num_obj > 0 and
                                          not self.object_manager.has_all(objects))
        ms_features, key, shrinkage, selection = self._features(image_ti, image)
        if need_segment:
            prob = self._segment(key, selection, ms_features, update_sensory=not end)

        if mask is not None:
            tmp_ids, _ = self.object_manager.add_new_objects(objects)
            mask, _ = pad_divide_by(mask, 16)
            if need_segment:
                # the given mask overrides the prediction where it is set (mutual exclusivity)
                no_bg = prob[1:]
                taken = (mask > 0) if hard_mask else (mask.max(0)[0] > 0.5)
                no_bg[:, taken] = 0
                fresh = []
                for j, tmp in enumerate(tmp_ids):
                    this = (mask == objects[j]).type_as(no_bg) if hard_mask else mask[tmp]
                    if tmp >= no_bg.shape[0]:
                        fresh.append(this.unsqueeze(0))
                    else:
                        no_bg[tmp + 1] = this
                mask = torch.cat([no_bg, *fresh], dim=0)
            elif hard_mask:
                mask = torch.stack([mask == objects[j] for j in range(len(tmp_ids))], dim=0)
            prob = torch.softmax(self.network.aggregate(mask, dim=0), dim=0)

        self.last_mask = prob[1:].unsqueeze(0)
        if is_mem_frame:
            self._add_memory(image, ms_features, self.last_mask, key, shrinkage, selection)
        if delete_buffer:
            self.image_feature_store.delete(image_ti)
        return unpad(prob, self.pad)
