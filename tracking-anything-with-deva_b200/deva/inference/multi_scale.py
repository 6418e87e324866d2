"""Multi-scale / flip test-time augmentation in one pass (evaluation/eval_vos.py with ``--size``, ``--flip`` and
``--save_scores``, then scripts/merge_multi_scale.py), with the score export and the merge on the device.

The reference runs eval_vos once per member (each with its own working size, flipped or not), dumps every frame's
resized-back probabilities as ``(prob * 255).astype(np.uint8)``, and merges the dumps offline: float32 sum over the
members, ``np.argmax`` over channels, remap through the ``{object id: tmp id}`` dict.  ``MultiScaleCore`` runs the
members side by side over one stream of uint8 frames: per member the reader's resize (and the driver's flip) at
ingest, the member's ``step``, and ``prob_to_scores`` adding the member's scores into one int32 sum at the original
size; the merged id map comes from ``scores_to_ids``.  Nothing goes through the host.
"""
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from deva.inference.frame_io import (_to_device, frame_from_rgb8, mask_from_index8, prob_to_scores, scores_to_ids)
from deva.inference.inference_core import DEVAInferenceCore

Member = Tuple[Optional[int], bool]


def validate_members(members: Sequence) -> List[Member]:
    """``members`` -> list of (size, flip): size None (the native size, eval_vos' ``--size -1``) or a positive int
    (the short side, as the readers' ``Resize(size)``), flip a bool.  Raises ValueError on anything else."""
    out = []
    for m in members:
        try:
            size, flip = m
        except (TypeError, ValueError):
            raise ValueError(f'multi-scale member {m!r} is not a (size, flip) pair') from None
        if size is not None and (isinstance(size, bool) or not isinstance(size, int) or size <= 0):
            raise ValueError(f'multi-scale member {m!r}: size must be None or a positive int')
        if not isinstance(flip, bool):
            raise ValueError(f'multi-scale member {m!r}: flip must be a bool')
        out.append((size, flip))
    if not out:
        raise ValueError('multi-scale: no members')
    return out


class MultiScaleCore:
    """One ``DEVAInferenceCore`` per member (size, flip), all sharing ``network``; ``step`` feeds a frame to every
    member in order on the current stream and returns the merged id map at the frame's size."""

    def __init__(self, network, config: Dict, members: Sequence[Member]):
        self.members = validate_members(members)
        self.network = network
        self.cores = [DEVAInferenceCore(network, dict(config)) for _ in self.members]

    @property
    def object_manager(self):
        return self.cores[0].object_manager

    def step(self, frame_u8: torch.Tensor, mask_u8: Optional[torch.Tensor] = None, objects: Optional[List[int]] = None,
             *, end: bool = False,
             return_scores: bool = False) -> Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]]:
        """frame_u8 uint8 [H0, W0, 3] (host - ideally pinned - or device); mask_u8 uint8 [H0, W0] index mask with the
        ``objects`` it labels (required with a mask, so the mask is never read on the host).

        Returns the merged ids uint8 [H0, W0] (object ids; ids above 255 wrap), and with ``return_scores`` also the
        summed scores int32 [K+1, H0, W0].  Raises RuntimeError when members disagree on the channel count or on the
        temporary-id mapping: the reference's merge applies one mapping to every member."""
        if mask_u8 is not None and objects is None:
            raise ValueError('MultiScaleCore.step: a mask needs its objects')
        frame_u8 = _to_device(frame_u8, None)
        h0, w0 = frame_u8.shape[:2]
        if mask_u8 is not None:
            mask_u8 = _to_device(mask_u8, frame_u8.device)
            if tuple(mask_u8.shape) != (h0, w0):
                raise ValueError(f'MultiScaleCore.step: mask {tuple(mask_u8.shape)} for a {h0}x{w0} frame')
        total, mapping = None, None
        for i, ((size, flip), core) in enumerate(zip(self.members, self.cores)):
            image = frame_from_rgb8(frame_u8, size=size, resize='reader', flip=flip)
            if mask_u8 is None:
                prob = core.step(image, end=end)
            else:
                prob = core.step(image, mask_from_index8(mask_u8, size, flip=flip), objects, end=end)
            this_mapping = core.object_manager.get_tmp_to_obj_mapping()
            if total is None:
                total = torch.zeros(prob.shape[0], h0, w0, dtype=torch.int32, device=frame_u8.device)
                mapping = this_mapping
            elif prob.shape[0] != total.shape[0]:
                raise RuntimeError(f'multi-scale member {i} {self.members[i]} has {prob.shape[0]} channels, member 0 '
                                   f'has {total.shape[0]}')
            elif this_mapping != mapping:
                raise RuntimeError(f'multi-scale member {i} {self.members[i]} maps objects to temporary ids as '
                                   f'{this_mapping}, member 0 as {mapping}')
            prob_to_scores(prob.float(), size=(h0, w0), flip=flip, scores=False, into=total)
        ids = scores_to_ids(total, mapping=mapping)
        return (ids, total) if return_scores else ids
