"""Stuff merging of VIPSeg predictions (the reference's deva/vps_metrics/stuff_merging.py) with the id rewrite on the
device.

Per video, IDPostprocessor's rules run on the host over the JSON entries alone: a thing whose category changes gets a
new id, every stuff category maps to one id, and a collision draws from the global ``np.random`` as the reference does.
That gives each frame a table -> output-id rewrite, which ``deva_b200_pano_remap`` applies per pixel while it writes the
RGB of the new id and counts the pixels of every output id (the areas that decide which stuff entries are kept).  PNGs
are decoded and encoded on a pool of host threads; with ``png_encoder='device'`` (or ``DEVA_B200_PNG_ENCODER=device``)
the rewritten maps are encoded on the device (deva/utils/png_encode.py) and only the compressed files come back; with
``png_decoder='device'`` (or ``DEVA_B200_PNG_DECODER=device``) the input maps are decoded on the device
(deva/utils/png_decode.py) and only the compressed files go up.

Videos are processed in order in this process.  The reference maps them over ``Pool(16)``, so its random draws depend on
which worker handles which video; here they follow the order of ``pred.json``, as a serial run of the reference's
``process_single_video`` does.
"""
import json
import os
from os import path

import numpy as np
import torch
from PIL import Image

from deva.utils.device_download import write
from deva.utils.png_decode import resolve_decoder
from deva.utils.png_encode import encode_png_async, resolve_encoder
from deva.vps_metrics import scoring, video_pass


def _save(rgb: np.ndarray, file: str):
    Image.fromarray(rgb).save(file)


def merge_stuff(input_path, output_path, isthing=None, num_threads=None, *, png_encoder=None, png_decoder=None):
    """isthing: {category id: bool}; None = the VIPSeg category table (deva.utils.pano_utils.vipseg_cat_to_isthing,
    which comes from the reference checkout).  png_encoder: 'pil' or 'device'; None reads DEVA_B200_PNG_ENCODER
    (default 'pil').  png_decoder: 'pil' or 'device'; None reads DEVA_B200_PNG_DECODER (default 'pil')."""
    png_encoder = resolve_encoder(png_encoder)
    png_decoder = resolve_decoder(png_decoder)
    if isthing is None:
        from deva.utils.pano_utils import vipseg_cat_to_isthing as isthing
    from deva import _native
    with open(path.join(input_path, 'pred.json')) as f:
        annotations = json.load(f)['annotations']
    dev = video_pass.require_device()
    decoder, upload = video_pass.make_decoder(png_decoder, dev, num_threads), video_pass.Uploader(dev)
    writes = []
    output_annotations = []
    try:
        for vid_ann in annotations:
            video_id = vid_ann['video_id']
            out_dir = path.join(output_path, 'pan_pred', video_id)
            os.makedirs(out_dir, exist_ok=True)
            table, frames, _ = scoring.merge_plan(vid_ann, isthing)
            names = [ann['file_name'].replace('.jpg', '.png') for ann in vid_ann['annotations']]
            ids = torch.from_numpy(table).to(dev)
            n_out = max([len(f[1]) for f in frames] + [1])
            counts = torch.empty(len(frames), n_out, dtype=torch.int32, device=dev)
            unknown = torch.empty(len(frames), 1, dtype=torch.int32, device=dev)
            outs = []
            for t, mask in enumerate(decoder.frames([path.join(input_path, 'pan_pred', video_id, n) for n in names])):
                slot, out_ids, _, _ = frames[t]
                out = torch.empty(mask.shape, dtype=torch.uint8, device=dev)
                _native.pano_remap(upload(mask), ids, torch.from_numpy(slot).to(dev, non_blocking=True),
                                   torch.from_numpy(out_ids).to(dev, non_blocking=True), out,
                                   counts[t, :len(out_ids)], unknown[t])
                outs.append(encode_png_async(out, 'RGB') if png_encoder == 'device' else out)
            counts_h = counts.cpu().numpy()
            video_annotations = []
            for t, (ann, (slot, out_ids, things, stuff_to_id)) in enumerate(zip(vid_ann['annotations'], frames)):
                segments = scoring.merged_segments(things, stuff_to_id, out_ids, counts_h[t, :len(out_ids)], isthing)
                video_annotations.append({'file_name': ann['file_name'], 'segments_info': segments})
                if png_encoder == 'device':
                    writes.append(decoder.pool.submit(write, outs[t], path.join(out_dir, names[t])))
                else:
                    writes.append(decoder.pool.submit(_save, outs[t].cpu().numpy(), path.join(out_dir, names[t])))
            output_annotations.append({'video_id': video_id, 'annotations': video_annotations})
        for w in writes:
            w.result()
    finally:
        decoder.close()
    with open(path.join(output_path, 'pred.json'), 'w') as f:
        json.dump({'annotations': output_annotations}, f)
