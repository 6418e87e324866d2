"""Mint the resized-ingest fixtures (SURVEY 8f-3) from the UNMODIFIED reference on the CPU (build container only).

    python tests/golden/make_ingest_golden.py

Reuses make_golden.py's shims and helpers by importing it (nothing of make_golden runs but its module set-up) and
writes only ingest_vos240.{npz,json} and ingest_vipseg.npz, so every other fixture stays byte-identical.

(1) example/vos/bmx-trees through evaluation/eval_vos.py:133-198 at --size 240 (854x480 -> 427x240), with and without
--flip: the reader's own im_transform / mask_transform (video_reader.py:140-161; pycocotools, which the reader imports
for a path not taken here, is stubbed), the flip, step, the resize back to 480x854, the flip back, argmax and
tmp_to_obj_cls.  Stored like config1_vos.npz (per frame the id map and the confident-pixel mask of the resized-back
probabilities), with the step's probabilities on a stride-8 lattice, plus the reader's first-frame mask and its resized
first frame on the same lattice.  The uint8 frames are config1_vos.npz's frames_u8.
(2) One example/vipseg frame (1280x720) through the reader convention (Resize(480, BILINEAR, antialias=True)) and the
demo convention (demo_utils.get_input_frame_for_deva(frame, 480), its .cuda() left out).  Stored: the JPEG file as is
(a fraction of the decoded frame's size), a stride-16 lattice of its PIL decode to confirm the decoder, and both
outputs on a stride-8 lattice with their full shapes.
"""
import io
import json
import os
import sys
import types

sys.dont_write_bytecode = True
import make_golden as mg  # noqa: E402  (sets up the reference import and its shims)

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image

LATTICE = 8


def ingest_vos240():
    coco = types.ModuleType('pycocotools')
    coco.mask = types.ModuleType('pycocotools.mask')
    sys.modules['pycocotools'], sys.modules['pycocotools.mask'] = coco, coco.mask
    from deva.inference.data.video_reader import VideoReader
    root, vid = '/root/reference/example/vos', 'bmx-trees'
    arrays = {}
    meta = {'size': 240, 'video': vid, 'lattice': LATTICE, 'runs': {}}
    for flip in (False, True):
        reader = VideoReader(vid, os.path.join(root, 'JPEGImages', vid), os.path.join(root, 'Annotations', vid), size=240)
        cfg = dict(mg.CFG)
        vid_length = len(reader)
        cfg['enable_long_term_count_usage'] = bool(cfg['enable_long_term'] and (
            vid_length / (cfg['max_mid_term_frames'] - cfg['min_mid_term_frames']) * cfg['num_prototypes']) >= cfg['max_long_term_elements'])
        net = mg.DEVA(cfg).eval()
        net.load_weights(mg.param_spec.synthetic_state_dict(seed=1))
        np.random.seed(42)
        core = mg.DEVAInferenceCore(net, cfg)
        tag = 'flip' if flip else 'noflip'
        for t in range(vid_length):
            data = reader[t]
            image, mask, labels = data['rgb'], data.get('mask'), data.get('valid_labels')
            if t == 0:
                assert mask is not None
                if not flip:
                    arrays['image0_lattice'] = image[:, ::LATTICE, ::LATTICE].contiguous()
                    arrays['image0_shape'] = np.array(image.shape)
                    arrays['mask0'] = mask.to(torch.uint8)
                meta['labels'] = labels.tolist()
            if flip:
                image = torch.flip(image, dims=[-1])
                mask = torch.flip(mask, dims=[-1]) if mask is not None else None
            prob = core.step(image, mask, labels.tolist() if labels is not None else None, end=(t == vid_length - 1))
            up = F.interpolate(prob.unsqueeze(1), tuple(int(v) for v in data['info']['shape']), mode='bilinear',
                               align_corners=False)[:, 0]
            if flip:
                up = torch.flip(up, dims=[-1])
            ids = core.object_manager.tmp_to_obj_cls(torch.argmax(up, dim=0))
            top2 = torch.topk(up, 2, dim=0)[0]
            arrays[f'{tag}_ids_{t}'] = ids.numpy().astype(np.uint8)
            arrays[f'{tag}_confident_{t}'] = np.packbits(((top2[0] - top2[1]) > 0.05).numpy())
            arrays[f'{tag}_prob_lattice_{t}'] = prob[:, ::LATTICE, ::LATTICE].contiguous().numpy()
            print('  ingest', tag, 't', t, 'prob', tuple(prob.shape), 'ids', np.unique(arrays[f'{tag}_ids_{t}']).tolist())
        meta['runs'][tag] = cfg
    mg.save('ingest_vos240.npz', **arrays)
    json.dump(meta, open(os.path.join(mg.HERE, 'ingest_vos240.json'), 'w'))


def ingest_vipseg():
    from deva.inference.data.video_reader import VideoReader
    sys.modules.setdefault('supervision', types.ModuleType('supervision'))  # result_utils' import, unused here
    from deva.inference.demo_utils import get_input_frame_for_deva
    vroot = '/root/reference/example/vipseg/images'
    vdir = os.path.join(vroot, sorted(os.listdir(vroot))[0])
    name = sorted(os.listdir(vdir))[0]
    jpeg = open(os.path.join(vdir, name), 'rb').read()
    frame = np.array(Image.open(io.BytesIO(jpeg)).convert('RGB'))
    reader = VideoReader('vipseg', vdir, vdir, size=480)  # only im_transform is used
    by_reader = reader.im_transform(Image.fromarray(frame))
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        by_demo = get_input_frame_for_deva(frame, 480)
    finally:
        torch.Tensor.cuda = cuda
    mg.save('ingest_vipseg.npz', jpeg=np.frombuffer(jpeg, np.uint8), decoded_lattice=frame[::16, ::16],
            reader_shape=np.array(by_reader.shape), reader_lattice=by_reader[:, ::LATTICE, ::LATTICE].contiguous(),
            demo_shape=np.array(by_demo.shape), demo_lattice=by_demo[:, ::LATTICE, ::LATTICE].contiguous())
    print('  vipseg', name, frame.shape, 'reader', tuple(by_reader.shape), 'demo', tuple(by_demo.shape))


if __name__ == '__main__':
    ingest_vos240()
    ingest_vipseg()
