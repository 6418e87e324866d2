"""Seeded synthetic VIPSeg-style dataset for the video panoptic metric fixtures, shared by make_vps_golden.py (reference
side), the oracle tests, the GPU tests and tools/bench_vps_metrics.py.  numpy + PIL only - imports nothing from the
reference, the product or the oracle.

write_dataset(root) writes
  root/truth/<video>/<frame>.png        ground-truth RGB id PNGs (id = r + 256 g + 65536 b)
  root/panoptic_gt.json                 {'categories', 'videos': [{'video_id', 'images'}], 'annotations'}
  root/submit/pan_pred/<video>/*.png    predictions, root/submit/pred.json
What the videos contain:
  * stuff bands (several predicted stuff segments of one category), things that drift, VOID margins;
  * a crowd segment, a ground-truth id painted but not listed, a listed ground-truth id with no pixels;
  * duplicate JSON entries (ground truth and prediction), ids >= 2^16;
  * a predicted thing whose category changes (stuff merging has to draw a new id);
  * in 'v_small' frame 0, a thing pair whose IoU is exactly 0.5; a false positive mostly on VOID;
  * a one-frame video, videos shorter and longer than 10 frames and one 720x1280 video.
"""
import json
import os

import numpy as np
from PIL import Image

N_CATEGORIES = 124
CATEGORIES = [{'id': c, 'name': f'class{c}', 'isthing': int(c % 4 == 0)} for c in range(N_CATEGORIES)]
ISTHING = {c['id']: c['isthing'] == 1 for c in CATEGORIES}
# video id -> (frames, h, w, things, seed)
VIDEOS = {'v_small': (6, 40, 56, 4, 1), 'v_one': (1, 30, 40, 3, 2), 'v_long': (12, 32, 48, 6, 3),
          'v_720p': (3, 720, 1280, 40, 4)}
MERGE_SEED = 7  # np.random.seed before stuff merging


def id_to_rgb(ids: np.ndarray) -> np.ndarray:
    return np.stack([(ids >> (8 * i)) & 255 for i in range(3)], axis=-1).astype(np.uint8)


def _entries(id_map, meta, dup=None):
    """JSON segments for the ids painted in id_map (in meta's order); dup: id listed twice with its area split."""
    ids, counts = np.unique(id_map, return_counts=True)
    area = dict(zip(ids.tolist(), counts.tolist()))
    out = []
    for sid, info in meta.items():
        if sid not in area and not info.get('keep_absent'):
            continue
        a = area.get(sid, 0)
        e = {'id': sid, 'category_id': info['category_id'], 'iscrowd': info.get('iscrowd', 0), 'area': a}
        if sid == dup and a > 1:
            out += [dict(e, area=a // 2), dict(e, area=a - a // 2)]
        else:
            out.append(e)
    return out


def make_video(name):
    """-> list of (gt id map int64, gt segments, pred id map, pred segments) per frame."""
    t_len, h, w, n_things, seed = VIDEOS[name]
    rng = np.random.default_rng(seed)
    stuff_cats = [c for c in range(N_CATEGORIES) if c % 4][:6]
    thing_cats = [c for c in range(N_CATEGORIES) if c % 4 == 0]
    n_bands = 3
    bands = np.linspace(0, h, n_bands + 1).astype(int)
    things = []
    for k in range(n_things):
        th, tw = int(rng.integers(h // 8 + 2, h // 3 + 3)), int(rng.integers(w // 8 + 2, w // 3 + 3))
        things.append(dict(y=float(rng.integers(0, h - th)), x=float(rng.integers(0, w - tw)), h=th, w=tw,
                           vy=float(rng.normal(0, 1)), vx=float(rng.normal(0, 1.5)),
                           gt_id=int(70000 + 131 * k if k % 2 == 0 else 300 + k),
                           pred_id=int(65536 * 3 + 17 * k if k % 3 == 1 else 5 + k),
                           cat=int(thing_cats[int(rng.integers(0, 4))]), crowd=(k == n_things - 1 and n_things > 2)))
    frames = []
    for t in range(t_len):
        gt = np.zeros((h, w), np.int64)
        pred = np.zeros((h, w), np.int64)
        gt_meta, pred_meta = {}, {}
        for b in range(n_bands):
            gid = 1000 + b
            gt[bands[b]:bands[b + 1], :w - 2] = gid  # the last two columns stay VOID
            gt_meta[gid] = {'category_id': stuff_cats[b]}
            # prediction: the band, shifted by one row, in two segments of the same category
            y0, y1 = max(bands[b] + 1, 0), min(bands[b + 1] + 1, h)
            half = w // 2 + (t % 3)
            pred[y0:y1, :half] = 10 + 2 * b
            pred[y0:y1, half:] = 11 + 2 * b
            pred_meta[10 + 2 * b] = {'category_id': stuff_cats[b]}
            pred_meta[11 + 2 * b] = {'category_id': stuff_cats[b]}
        for k, th in enumerate(things):
            y = int(np.clip(th['y'] + th['vy'] * t, 0, h - th['h']))
            x = int(np.clip(th['x'] + th['vx'] * t, 0, w - th['w']))
            gt[y:y + th['h'], x:x + th['w']] = th['gt_id']
            gt_meta[th['gt_id']] = {'category_id': th['cat'], 'iscrowd': int(th['crowd'])}
            if k == 1 and t % 4 == 3:
                continue  # missed detection
            jy, jx = int(rng.integers(-1, 2)), int(rng.integers(-1, 2))
            py, px = int(np.clip(y + jy, 0, h - th['h'])), int(np.clip(x + jx, 0, w - th['w']))
            pred[py:py + th['h'], px:px + th['w']] = th['pred_id']
            cat = th['cat']
            if k == 0 and t >= t_len // 2:
                cat = thing_cats[(thing_cats.index(cat) + 1) % len(thing_cats)]  # the category changes mid-video
            pred_meta[th['pred_id']] = {'category_id': cat}
        # a ground-truth id that is painted but not listed, and one listed without pixels
        gt[h - 3:h, 0:3] = 555
        gt_meta[777] = {'category_id': thing_cats[1], 'keep_absent': True}
        # a false positive lying mostly on the VOID margin
        pred[0:4, w - 3:w] = 99
        pred_meta[99] = {'category_id': thing_cats[2]}
        if name == 'v_small' and t == 0:
            # IoU exactly 0.5: gt 4x3 at (30, 40), pred 4x3 at (30, 41), intersection 8, union 16, no VOID inside
            gt[28:36, 38:46] = 1001
            pred[28:36, 38:46] = 12
            gt[30:34, 40:43] = 4242
            pred[30:34, 41:44] = 4243
            gt_meta[4242] = {'category_id': 8, 'iscrowd': 0}
            pred_meta[4243] = {'category_id': 8}
        gt_seg = _entries(gt, gt_meta, dup=things[0]['gt_id'] if t % 2 == 0 else None)
        pred_seg = _entries(pred, pred_meta, dup=10 if t % 2 == 1 else None)
        for e in pred_seg:
            del e['iscrowd']
        frames.append((gt, gt_seg, pred, pred_seg))
    return frames


def write_dataset(root):
    """Writes the dataset under root; -> (submit_dir, truth_dir, gt json path)."""
    truth, submit = os.path.join(root, 'truth'), os.path.join(root, 'submit')
    gt_json = {'categories': CATEGORIES, 'videos': [], 'annotations': []}
    pred_json = {'annotations': []}
    for name in VIDEOS:
        os.makedirs(os.path.join(truth, name), exist_ok=True)
        os.makedirs(os.path.join(submit, 'pan_pred', name), exist_ok=True)
        images, gt_anns, pred_anns = [], [], []
        for t, (gt, gt_seg, pred, pred_seg) in enumerate(make_video(name)):
            fname = f'{t:08d}.png'
            Image.fromarray(id_to_rgb(gt)).save(os.path.join(truth, name, fname))
            Image.fromarray(id_to_rgb(pred)).save(os.path.join(submit, 'pan_pred', name, fname))
            images.append({'file_name': fname, 'id': f'{name}_{t}'})
            gt_anns.append({'file_name': fname, 'segments_info': gt_seg})
            pred_anns.append({'file_name': fname, 'segments_info': pred_seg})
        gt_json['videos'].append({'video_id': name, 'images': images})
        gt_json['annotations'].append({'video_id': name, 'annotations': gt_anns})
        pred_json['annotations'].append({'video_id': name, 'annotations': pred_anns})
    gt_path = os.path.join(root, 'panoptic_gt.json')
    with open(gt_path, 'w') as f:
        json.dump(gt_json, f)
    with open(os.path.join(submit, 'pred.json'), 'w') as f:
        json.dump(pred_json, f)
    return submit, truth, gt_path


def break_prediction(submit_dir, kind):
    """Make the prediction of 'v_small' frame 1 invalid: 'png' drops a painted id from the JSON, 'json' lists an id the
    PNG does not have, 'unlisted' paints ids that no entry of the video lists (one of them VOID's neighbour 1, one
    >= 2^16).  Rewrites pred.json or the PNG in place."""
    if kind == 'unlisted':
        png = os.path.join(submit_dir, 'pan_pred', 'v_small', '00000001.png')
        rgb = np.array(Image.open(png))
        rgb[5:7, 5:9] = id_to_rgb(np.array([[424242]]))
        rgb[8, 20] = id_to_rgb(np.array([[1]]))
        Image.fromarray(rgb).save(png)
        return
    path = os.path.join(submit_dir, 'pred.json')
    with open(path) as f:
        pred = json.load(f)
    seg = pred['annotations'][0]['annotations'][1]['segments_info']
    if kind == 'png':
        victim = seg[2]['id']
        seg[:] = [e for e in seg if e['id'] != victim]
    else:
        seg += [{'id': 123456, 'category_id': 4, 'area': 1}, {'id': 31, 'category_id': 8, 'area': 1}]
    with open(path, 'w') as f:
        json.dump(pred, f)
