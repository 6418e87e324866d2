"""Mint tests/golden/sam_masks.{json,npz} from the UNMODIFIED reference SamAutomaticMaskGenerator
(deva/ext/SAM/automatic_mask_generator.py, staged under oracle/_ref by oracle/build_ref_sam.py), run on the CPU over
oracle/sam_stub.py's stand-in segment_anything and FakeSam, for every case of sam_masks_scenario.py.

    python tests/golden/make_sam_masks_golden.py

Per case the json holds the field dtypes and shapes, or the exception the reference raised; the npz holds iou_preds,
points, stability_score (as int32 bit patterns, so nan compares) and boxes, and the masks as the per-mask pixel count
and one sha256 of np.packbits over the whole bool array.
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import sam_masks_scenario as sc  # noqa: E402
from oracle import sam_masks, sam_stub  # noqa: E402


def digest(masks: torch.Tensor) -> str:
    return hashlib.sha256(np.packbits(masks.cpu().numpy().astype(np.uint8), axis=None).tobytes()).hexdigest()


def record(out):
    """MaskData / dict -> (json entry, npz arrays)."""
    masks = out['masks']
    meta = {k: [str(out[k].dtype).replace('torch.', ''), list(out[k].shape)]
            for k in ('masks', 'iou_preds', 'points', 'stability_score', 'boxes')}
    meta['mask_sha256'] = digest(masks)
    arrays = {'iou_preds': out['iou_preds'].cpu().numpy(), 'points': out['points'].cpu().numpy(),
              'stability_bits': out['stability_score'].cpu().contiguous().view(torch.int32).numpy(),
              'boxes': out['boxes'].cpu().numpy(), 'areas': masks.flatten(1).sum(1).cpu().numpy()}
    return meta, arrays


def main():
    Gen = sam_masks.reference_generator()
    meta, arrays = {}, {}
    for case in sc.CASES:
        mk, gk, img, pos, neg = sc.arguments(case)
        try:
            out = Gen(sam_stub.FakeSam(**mk), **gk).generate(img, pos, neg)
        except Exception as e:  # the reference's own failure is part of the record
            meta[case] = {'error': type(e).__name__}
            print(case, 'raises', type(e).__name__)
            continue
        m, a = record(out)
        meta[case] = m
        arrays.update({f'{case}/{k}': v for k, v in a.items()})
        print(case, m['masks'], m['boxes'][0], 'nan stability' if np.isnan(out['stability_score'].numpy()).any() else '')
    json.dump(meta, open(os.path.join(HERE, 'sam_masks.json'), 'w'), indent=1, sort_keys=True)
    np.savez_compressed(os.path.join(HERE, 'sam_masks.npz'), **arrays)


if __name__ == '__main__':
    main()
