"""Mint the detector-mask fixture from the UNMODIFIED reference on the CPU (build container only).

    python tests/golden/make_detector_masks_golden.py

Runs the reference's ``deva/ext/automatic_sam.py::auto_segment`` and ``deva/ext/grounding_dino.py::segment_with_text``
over detector_masks_scenario's cases, with stub ``segment_anything`` / ``groundingdino`` / ``deva.ext.SAM`` /
``MobileSAM`` / ``LightHQSAM`` modules and fakes that return seeded masks and record every call.  Writes
detector_masks.{json,npz}: id maps, segment lists, the recorded calls, and the getters' recorded model builds.

Automatic-path seeds are drawn until every output pixel's top two scored values (duplicate masks merged) differ by more
than 1e-4 relative and no resized value lies within 1e-5 of 0.5 without being 0.5, so the CPU-minted maps are the
device's maps too.
"""
import json
import os
import sys

sys.dont_write_bytecode = True
import make_golden as mg  # noqa: E402  (puts the reference on sys.path, with its shims)

import numpy as np
import torch
import torch.nn.functional as F

import detector_masks_scenario as sc

MARGIN = 1e-4


def auto_margin_ok(masks, out_hw, suppress):
    if masks.shape[0] == 0:
        return True
    _, first = np.unique(masks.reshape(masks.shape[0], -1), axis=0, return_index=True)
    v = F.interpolate(torch.from_numpy(masks).float()[None], out_hw, mode='bilinear')[0]
    area = v.flatten(1).sum(1)
    score = area if suppress else area.max() * 2 - area
    scored = torch.cat([torch.full((1, *out_hw), 0.1), (v * score[:, None, None])[np.sort(first)]])
    top = torch.topk(scored, min(2, scored.shape[0]), dim=0)[0]
    rel = ((top[0] - top[1]) / top[0]).min() if top.shape[0] == 2 else torch.tensor(1.)
    near = (v - 0.5).abs()
    near = near[near > 0]
    return float(rel) > MARGIN and (near.numel() == 0 or float(near.min()) > 1e-5)


def main():
    recorder = []
    sc.install_detector_stubs(recorder)
    from deva.ext import automatic_sam, grounding_dino  # the reference's modules
    assert automatic_sam.__file__.startswith('/root/reference'), automatic_sam.__file__
    meta = {'margin': MARGIN, 'auto': [], 'text': []}
    arrays = {}
    for i, (name, (h, w), min_side, suppress, thr, fwd, spec) in enumerate(sc.AUTO_CASES):
        seed = 1000 * (i + 1)
        out_hw = (int(h * min_side / min(h, w)), int(w * min_side / min(h, w))) if min_side > 0 else (h, w)
        while not auto_margin_ok(sc.build_masks(spec, h, w, seed), out_hw, suppress):
            seed += 1
        masks = sc.build_masks(spec, h, w, seed)
        sam = sc.FakeAutoSam(masks, sc.iou_preds(len(masks), seed), 'cpu')
        fm = sc.forward_mask(fwd, h, w)
        if fm is not None:  # positive-point labels well away from the 0.01 cut, so CUDA's blur selects the same
            fg = F.interpolate((fm > 0).float()[None, None], scale_factor=1 / 16, mode='bilinear', antialias=True)
            n = sc.POINTS_PER_SIDE
            side = torch.linspace(1 / (2 * n), 1 - 1 / (2 * n), n)
            pts = torch.stack([side[None].repeat(n, 1), side[:, None].repeat(1, n)], -1)[None]
            lab = F.grid_sample(fg, pts * 2 - 1, align_corners=False).view(-1)
            assert float((lab - 0.01).abs().min()) > 1e-3
        out, segs = automatic_sam.auto_segment(sc.auto_config(thr), sam, sc.image(h, w), fm, min_side, suppress)
        arrays[f'auto_{name}'] = out.numpy().astype(np.int16)
        meta['auto'].append({'name': name, 'seed': seed, 'segments': sc.segments_json(segs), 'calls': sam.calls})
        print(f'  auto {name}: seed {seed}, {len(masks)} masks -> {len(segs)} segments, map {tuple(out.shape)}')
    for name, (h, w), min_side, nms, boxes in sc.TEXT_CASES:
        gd, sam = sc.FakeGroundingDino(boxes, 'cpu'), sc.FakeSamPredictor()
        out, segs = grounding_dino.segment_with_text(sc.text_config(nms), gd, sam, sc.image(h, w), ['a', 'b'],
                                                     min_side)
        arrays[f'text_{name}'] = out.numpy().astype(np.int16)
        meta['text'].append({'name': name, 'segments': sc.segments_json(segs), 'calls': gd.calls + sam.calls})
        print(f'  text {name}: {len(boxes)} boxes -> {len(segs)} segments, map {tuple(out.shape)}')
    meta['model_builds'] = sc.record_model_builds(automatic_sam.get_sam_model, grounding_dino.get_grounding_dino_model,
                                                  recorder)
    mg.save('detector_masks.npz', **arrays)
    json.dump(meta, open(os.path.join(mg.HERE, 'detector_masks.json'), 'w'))


if __name__ == '__main__':
    main()
