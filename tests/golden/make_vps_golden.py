"""Mint the video panoptic metric fixture from the UNMODIFIED reference on the CPU (build container only).

    python tests/golden/make_vps_golden.py

On the dataset of vps_scenario.write_dataset it runs the reference's
  * stuff merging: ``process_single_video`` called serially over pred.json's videos after ``np.random.seed(MERGE_SEED)``,
    with the scenario's category table in place of VIPSeg's (its ``merge_stuff`` maps the videos over Pool(16));
  * ``vpq_compute_single_core`` for every video and window size (the per-category stats, summed video by video), and
    ``eval_vpq`` itself for the text files;
  * ``eval_stq`` (its ``STQuality`` captured for the result values) for stq.txt;
  * both prediction KeyErrors, on copies broken by vps_scenario.break_prediction (the 'png not json' one twice: an id
    listed in another frame, and ids that no entry of the video lists).
Writes vps_metrics.json (floats as float.hex, merged PNG pixels as sha256, text files verbatim) and vps_metrics.npz
(the merged id images of the small videos).
"""
import copy
import hashlib
import json
import os
import shutil
import sys
import tempfile

sys.dont_write_bytecode = True
import make_golden as mg  # noqa: E402  (puts the reference first on sys.path, with its shims)

import numpy as np  # noqa: E402
from PIL import Image  # noqa: E402

import vps_scenario as vs  # noqa: E402
import deva.vps_metrics.eval_stq_vipseg as es  # noqa: E402
import deva.vps_metrics.eval_vpq_vipseg as ev  # noqa: E402
import deva.vps_metrics.stuff_merging as sm  # noqa: E402

assert ev.__file__.startswith('/root/reference'), ev.__file__


def gt_pred_split(submit, truth, gt_path):
    gt_jsons = json.load(open(gt_path))
    pred_j = {a['video_id']: a['annotations'] for a in json.load(open(os.path.join(submit, 'pred.json')))['annotations']}
    gt_j = {a['video_id']: a['annotations'] for a in gt_jsons['annotations']}
    out = []
    for video in gt_jsons['videos']:
        vid = video['video_id']
        names = [im['file_name'] for im in video['images']]
        out.append(list(zip(gt_j[vid], pred_j[vid], [os.path.join(truth, vid, n) for n in names],
                            [os.path.join(submit, 'pan_pred', vid, n) for n in names], video['images'])))
    return {el['id']: el for el in gt_jsons['categories']}, out


def stat_json(stat):
    return {str(k): [float(v.iou).hex(), int(v.tp), int(v.fp), int(v.fn)] for k, v in stat.pq_per_cat.items()}


def main():
    meta, arrays = {'isthing': {str(k): v for k, v in vs.ISTHING.items()}, 'merge_seed': vs.MERGE_SEED}, {}
    with tempfile.TemporaryDirectory() as root:
        submit, truth, gt_path = vs.write_dataset(root)
        # stuff merging
        merged = os.path.join(root, 'merged')
        sm.vipseg_cat_to_isthing = vs.ISTHING
        np.random.seed(vs.MERGE_SEED)
        anns = json.load(open(os.path.join(submit, 'pred.json')))['annotations']
        meta['merged_json'] = {'annotations': [sm.process_single_video(a, submit, merged) for a in anns]}
        meta['merged_sha256'] = {}
        for a in anns:
            for t, f in enumerate(a['annotations']):
                px = np.array(Image.open(os.path.join(merged, 'pan_pred', a['video_id'], f['file_name'])))
                meta['merged_sha256'][f"{a['video_id']}/{f['file_name']}"] = hashlib.sha256(px.tobytes()).hexdigest()
                if px.size < 100000:
                    arrays[f"merged_{a['video_id']}_{t}"] = px
        # VPQ: per-video stats for every window size, then the reference's own eval_vpq for the files
        categories, split = gt_pred_split(submit, truth, gt_path)
        meta['vpq_stats'] = {}
        for n in (1, 2, 4, 6, 8, 10, 999):
            total = ev.PQStat()
            per_video = []
            for video in copy.deepcopy(split):
                s = ev.vpq_compute_single_core(categories, n, video)
                per_video.append(stat_json(s))
                total += s
            meta['vpq_stats'][str(n)] = {'total': stat_json(total), 'per_video': per_video}
        ev.eval_vpq(submit, truth, gt_path, num_processes=1)
        # STQ
        captured = []

        class Capture(es.numpy_stq.STQuality):
            def __init__(self, *a):
                super().__init__(*a)
                captured.append(self)

        es.numpy_stq.STQuality = Capture
        es.eval_stq(submit, truth, gt_path)
        r = captured[0].result()
        meta['stq'] = {'STQ': float(r['STQ']).hex(), 'AQ': float(r['AQ']).hex(), 'IoU': float(r['IoU']).hex(),
                       'AQ_per_seq': [float(v).hex() for v in r['AQ_per_seq']],
                       'IoU_per_seq': [float(v).hex() for v in r['IoU_per_seq']],
                       'Length_per_seq': [int(v) for v in r['Length_per_seq']]}
        meta['files'] = {name: open(os.path.join(submit, name)).read() for name in sorted(os.listdir(submit))
                         if name.endswith('.txt')}
        # the two prediction KeyErrors
        meta['errors'] = {}
        for kind in ('png', 'json', 'unlisted'):
            broken = os.path.join(root, f'broken_{kind}')
            shutil.copytree(submit, broken)
            vs.break_prediction(broken, kind)
            categories, split = gt_pred_split(broken, truth, gt_path)
            try:
                ev.vpq_compute_single_core(categories, 1, split[0])
                raise AssertionError('no KeyError')
            except KeyError as e:
                meta['errors'][kind] = e.args[0]
    mg.save('vps_metrics.npz', **arrays)
    json.dump(meta, open(os.path.join(mg.HERE, 'vps_metrics.json'), 'w'), indent=0)
    print('files:', sorted(meta['files']), 'errors:', meta['errors'])
    print('stq', meta['files']['stq.txt'].strip(), 'vpq-simple', meta['files']['vpq-simple.txt'])


if __name__ == '__main__':
    main()
