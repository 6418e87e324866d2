"""numpy restatement of VIPSeg's video panoptic metrics and stuff merging from per-frame joint label histograms.

The histograms are counted here with numpy (np.bincount over the pair of table indices) instead of
``deva_b200_pano_joint_hist``, and the rewrite of stuff merging with a table lookup instead of ``deva_b200_pano_remap``;
everything after the pixels - VPQ windows as prefix-sum differences, STQ's regrouping of cells, IDPostprocessor's rules -
is the package's host code (``deva.vps_metrics.scoring``, numpy only).  Checked against the unmodified reference's
outputs in tests/golden/vps_metrics.{json,npz}, this proves the histogram decomposition without a GPU.
"""
import json
import os

import numpy as np

from deva.vps_metrics import scoring, video_pass


def decode(rgb: np.ndarray) -> np.ndarray:
    rgb = rgb.astype(np.int64)
    return rgb[:, :, 0] + 256 * rgb[:, :, 1] + 65536 * rgb[:, :, 2]


def table_index(ids: np.ndarray, table: np.ndarray) -> np.ndarray:
    """Index of every id in the sorted table, len(table) when absent."""
    i = np.searchsorted(table, ids)
    found = (i < len(table)) & (table[np.minimum(i, len(table) - 1)] == ids) if len(table) else np.zeros(ids.shape, bool)
    return np.where(found, i, len(table))


def joint_hist(gt_rgb, pred_rgb, gt_ids, pred_ids) -> np.ndarray:
    cols = len(pred_ids) + 1
    code = table_index(decode(gt_rgb), gt_ids) * cols + table_index(decode(pred_rgb), pred_ids)
    return np.bincount(code.ravel(), minlength=(len(gt_ids) + 1) * cols).reshape(len(gt_ids) + 1, cols)


def histograms(decoder, gt_paths, pred_paths, gt_ids, pred_ids):
    return np.stack([joint_hist(video_pass.read_rgb(g), video_pass.read_rgb(p), gt_ids, pred_ids)
                     for g, p in zip(gt_paths, pred_paths)])


def evaluate(submit_dir, truth_dir, pan_gt_json_file):
    """-> ({nframes: PQStat}, STQuality, categories list)."""
    return video_pass.evaluate(submit_dir, truth_dir, pan_gt_json_file, num_threads=1, histograms=histograms)


def merge_stuff(input_path, isthing):
    """-> (output json, {'<video>/<file>': merged uint8 [h, w, 3]}); videos in order, np.random as seeded by the caller."""
    with open(os.path.join(input_path, 'pred.json')) as f:
        annotations = json.load(f)['annotations']
    out_json, images = [], {}
    for vid_ann in annotations:
        table, frames, _ = scoring.merge_plan(vid_ann, isthing)
        video_annotations = []
        for ann, (slot, out_ids, things, stuff_to_id) in zip(vid_ann['annotations'], frames):
            name = ann['file_name'].replace('.jpg', '.png')
            pred = video_pass.read_rgb(os.path.join(input_path, 'pan_pred', vid_ann['video_id'], name))
            s = slot[table_index(decode(pred), table)]
            counts = np.bincount(s.ravel(), minlength=len(out_ids))
            out = out_ids[s].astype(np.int64)
            images[f"{vid_ann['video_id']}/{name}"] = np.stack([(out >> (8 * i)) & 255 for i in range(3)], -1).astype(
                np.uint8)
            video_annotations.append({'file_name': ann['file_name'],
                                      'segments_info': scoring.merged_segments(things, stuff_to_id, out_ids, counts,
                                                                               isthing)})
        out_json.append({'video_id': vid_ann['video_id'], 'annotations': video_annotations})
    return {'annotations': out_json}, images
