"""Mint the multi-scale / flip fixture from the UNMODIFIED reference on the CPU (build container only).

    python tests/golden/make_multiscale_golden.py

Reuses make_golden.py's shims and helpers by importing it (nothing of make_golden runs but its module set-up) and
writes only multiscale_vos.{npz,json}, so every other fixture stays byte-identical.

(1) Members: example/vos/bmx-trees (854x480, synthetic checkpoint seed 1) through evaluation/eval_vos.py:133-211 with
--save_scores, once per member of sizes {240, 360, 480} x flip {off, on} (at 480 the reader's resize is the identity):
the reader's own transforms (pycocotools, which the reader imports for a path not taken here, is stubbed), the flip,
step, the resize back to 480x854, the flip back and ``(prob.cpu().numpy() * 255).astype(np.uint8)``.  The reference's
``ObjectManager.get_tmp_to_obj_mapping`` (object_manager.py:119-121) swaps its loop variables and raises, so eval_vos
cannot write backward.hkl at this commit; the mapping is computed as its intent, ``{obj.id: tmp}`` over
``tmp_id_to_obj``.
(2) Merge: the unmodified scripts/merge_multi_scale.py::process_vid over these arrays, with ``hickle`` stubbed by an
in-memory dict (the score directories hold empty placeholder files, which is all process_vid lists), its module
globals (all_options, args, out_path, palette) set as its __main__ would, and its palette PNGs read back.

Stored (npz): per member and frame the uint8 scores on a stride-8 lattice; per frame the merged id map in full; the
packed "decided" mask, where the top-two margin of the summed scores exceeds 2 * M (M members, each off by at most
1, cannot flip the argmax there); the summed scores on the lattice.  (json): members, config, labels, mapping.  The
uint8 frames and first-frame mask are config1_vos.npz's frames_u8 / mask0.
"""
import importlib.util
import json
import os
import sys
import tempfile
import types

sys.dont_write_bytecode = True
import make_golden as mg  # noqa: E402  (sets up the reference import and its shims)

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image, ImagePalette

LATTICE = 8
MEMBERS = [(size, flip) for size in (240, 360, 480) for flip in (False, True)]
ROOT, VID = '/root/reference/example/vos', 'bmx-trees'


def run_member(size, flip):
    """eval_vos.py:133-211 for one member -> (per-frame uint8 scores, frame names, mapping, labels, config)."""
    from deva.inference.data.video_reader import VideoReader
    reader = VideoReader(VID, os.path.join(ROOT, 'JPEGImages', VID), os.path.join(ROOT, 'Annotations', VID), size=size)
    cfg = dict(mg.CFG)
    vid_length = len(reader)
    cfg['enable_long_term_count_usage'] = bool(cfg['enable_long_term'] and (
        vid_length / (cfg['max_mid_term_frames'] - cfg['min_mid_term_frames']) * cfg['num_prototypes']) >= cfg['max_long_term_elements'])
    net = mg.DEVA(cfg).eval()
    net.load_weights(mg.param_spec.synthetic_state_dict(seed=1))
    np.random.seed(42)
    core = mg.DEVAInferenceCore(net, cfg)
    scores, names, labels = [], [], None
    for t in range(vid_length):
        data = reader[t]
        image, mask, valid = data['rgb'], data.get('mask'), data.get('valid_labels')
        if valid is not None:
            labels = valid.tolist()
        if flip:
            image = torch.flip(image, dims=[-1])
            mask = torch.flip(mask, dims=[-1]) if mask is not None else None
        prob = core.step(image, mask, valid.tolist() if valid is not None else None, end=(t == vid_length - 1))
        if data['info']['need_resize']:
            prob = F.interpolate(prob.unsqueeze(1), tuple(int(v) for v in data['info']['shape']), mode='bilinear',
                                 align_corners=False)[:, 0]
        if flip:
            prob = torch.flip(prob, dims=[-1])
        scores.append((prob.detach().cpu().numpy() * 255).astype(np.uint8))
        names.append(data['info']['frame'])
        print('  member', size, 'flip' if flip else 'noflip', 't', t, 'prob', tuple(prob.shape))
    # the intent of get_tmp_to_obj_mapping (object_manager.py:119-121), which raises as written
    mapping = {int(obj.id): int(tmp) for tmp, obj in core.object_manager.tmp_id_to_obj.items()}
    return scores, names, mapping, labels, cfg


def merge(per_member, names, mapping):
    """scripts/merge_multi_scale.py::process_vid, unmodified, over in-memory arrays -> per-frame id maps."""
    store = {}
    hickle = types.ModuleType('hickle')
    hickle.load = lambda p: store[os.path.realpath(p)]
    hickle.dump = lambda obj, p, **kw: store.__setitem__(os.path.realpath(p), obj)
    sys.modules['hickle'] = hickle
    spec = importlib.util.spec_from_file_location('merge_multi_scale', '/root/reference/scripts/merge_multi_scale.py')
    mms = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mms)
    from deva.utils.palette import davis_palette
    with tempfile.TemporaryDirectory() as tmp:
        options = []
        for m, scores in enumerate(per_member):
            d = os.path.join(tmp, f'member{m}', 'Scores')
            os.makedirs(os.path.join(d, VID))
            for name, s in zip(names, scores):
                p = os.path.join(d, VID, name[:-4] + '.hkl')
                open(p, 'wb').close()
                hickle.dump(s, p)
            p = os.path.join(d, VID, 'backward.hkl')
            open(p, 'wb').close()
            hickle.dump(mapping, p)
            options.append(d)
        out = os.path.join(tmp, 'merged')
        mms.all_options = options
        mms.args = types.SimpleNamespace(dataset='D')
        mms.out_path = out
        mms.palette = ImagePalette.ImagePalette(mode='P', palette=davis_palette)
        mms.process_vid(VID)
        return [np.array(Image.open(os.path.join(out, VID, name[:-4] + '.png'))) for name in names]


def multiscale_vos():
    coco = types.ModuleType('pycocotools')
    coco.mask = types.ModuleType('pycocotools.mask')
    sys.modules['pycocotools'], sys.modules['pycocotools.mask'] = coco, coco.mask
    per_member, names, mapping, labels, cfg = [], None, None, None, None
    for size, flip in MEMBERS:
        scores, names_m, mapping_m, labels_m, cfg_m = run_member(size, flip)
        assert names is None or (names_m == names and mapping_m == mapping and labels_m == labels and cfg_m == cfg)
        per_member.append(scores)
        names, mapping, labels, cfg = names_m, mapping_m, labels_m, cfg_m
    ids = merge(per_member, names, mapping)
    T = len(names)
    total = np.stack([sum(m[t].astype(np.float32) for m in per_member) for t in range(T)])  # [T, K+1, H, W]
    top2 = -np.sort(-total, axis=1)[:, :2]
    decided = (top2[:, 0] - top2[:, 1]) > 2 * len(MEMBERS)
    for t in range(T):
        print('  merged t', t, 'ids', np.unique(ids[t]).tolist(), f'decided {decided[t].mean():.4f}')
    mg.save('multiscale_vos.npz',
            scores_lattice=np.stack([np.stack([s[:, ::LATTICE, ::LATTICE] for s in m]) for m in per_member]),
            ids=np.stack(ids).astype(np.uint8),
            decided=np.packbits(decided),
            sum_lattice=total[:, :, ::LATTICE, ::LATTICE].astype(np.uint16))  # at most 6 * 255
    meta = {'video': VID, 'frames': names, 'members': [[s, f] for s, f in MEMBERS], 'lattice': LATTICE,
            'margin_per_member': 1, 'shape': list(ids[0].shape), 'labels': labels,
            'mapping': {str(k): v for k, v in mapping.items()}, 'config': cfg}
    json.dump(meta, open(os.path.join(mg.HERE, 'multiscale_vos.json'), 'w'))


if __name__ == '__main__':
    multiscale_vos()
