"""Mint the result-saver fixture from the UNMODIFIED reference on the CPU (build container only).

    python tests/golden/make_saver_golden.py

Reuses make_golden.py's shims by importing it and writes only saver.{json,npz}, so every other fixture stays
byte-identical.  The reference's own ``ResultSaver`` (deva/inference/result_utils.py) runs every session of
saver_session.SESSIONS - each dataset mode, need_resize on and off (also positional), long and short ids, prompts,
save_the_mask=False, path_to_image, objects added and deleted between frames (tmp ids repacked while earlier frames are
still queued) and a run longer than the product's pinned-buffer ring - with ``pycocotools`` / ``supervision`` stubbed
by recorders and ``PIL.Image.Image.save`` recording (path, mode, palette, pixels) instead of encoding.

Each frame's probabilities come from a seed; seeds are drawn until every output pixel's top-two margin after the CPU
interpolation exceeds 1e-4, so no near-tie can make a device id map differ.  The chosen seeds and the recordings are
stored.
"""
import json
import os
import sys
import tempfile

sys.dont_write_bytecode = True
import make_golden as mg  # noqa: E402  (sets up the reference import and its shims)

import numpy as np
import torch
import torch.nn.functional as F

import saver_session as ss

MARGIN = 1e-4


def margin(prob: np.ndarray, resize: bool) -> float:
    p = torch.from_numpy(prob)
    if resize:
        p = F.interpolate(p.unsqueeze(1), ss.OUT, mode='bilinear', align_corners=False)[:, 0]
    top2 = torch.topk(p, 2, dim=0)[0]
    return float((top2[0] - top2[1]).min())


def choose_seeds(index, session):
    """Per frame (prob seed, image seed), prob seeds drawn until the margin holds."""
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    om = ObjectManager()
    om.use_long_id = session[1]
    seeds = []
    for t, (ops, kw) in enumerate(session[4]):
        for op, arg in ops:
            if op == 'add':
                om.add_new_objects([ObjectInfo(i, category_id=c, score=s) for i, c, s in arg])
            else:
                om.delete_object(arg)
        seed = 1000 * (100 * index + t)
        while margin(ss.make_prob(seed, om.num_obj + 1), kw.get('resize') in (True, 'positional')) <= MARGIN:
            seed += 1
        seeds.append((seed, 7 * seed + 1))
    return seeds


def main():
    rec = ss.Recorder()
    meta, arrays = {'margin': MARGIN, 'sessions': []}, {}
    with rec.installed() as orig_save:
        from deva.inference import result_utils  # the reference's module: imports pycocotools / supervision eagerly
        from deva.inference.object_info import ObjectInfo
        from deva.inference.object_manager import ObjectManager
        assert result_utils.__file__.startswith('/root/reference'), result_utils.__file__
        for i, session in enumerate(ss.SESSIONS):
            seeds = choose_seeds(i, session)
            rec.events = []
            with tempfile.TemporaryDirectory() as root:
                video_json = ss.drive(result_utils.ResultSaver, ObjectManager, ObjectInfo, session, seeds, root, rec,
                                      orig_save)
            events = []
            for j, ev in enumerate(rec.events):
                key = f's{i}_e{j}'
                if isinstance(ev[-1], np.ndarray):
                    arrays[key] = ev[-1]
                    events.append(list(ev[:-1]) + [key])
                else:
                    events.append(list(ev))
            meta['sessions'].append({'seeds': seeds, 'video_json': video_json, 'events': events})
            kinds = [e[0] for e in events]
            print(f'  session {i} {session[0]} long={session[1]}: {len(session[4])} frames,',
                  {k: kinds.count(k) for k in sorted(set(kinds))})
    mg.save('saver.npz', **arrays)
    json.dump(meta, open(os.path.join(mg.HERE, 'saver.json'), 'w'))


if __name__ == '__main__':
    main()
