"""Mint the demo fixture from the UNMODIFIED reference on the CPU (build container only).

    python tests/golden/make_demo_golden.py

Reuses make_golden.py's shims (nothing of make_golden runs but its module set-up) and, like make_ingest_golden.py,
leaves out the reference's ``.cuda()``: ``Tensor.cuda`` is the identity while minting.  Writes demo.{json,npz}:

* the reference ``SimpleVideoReader``'s items over demo_scenario's reader folder and demo clip (names, order, SHA-256 of
  each array, errors);
* the reference ``get_input_frame_for_deva`` output for three small frames at each of INGEST_MIN_SIDES, whole;
* the reference demo loop (``DataLoader(reader, batch_size=None, collate_fn=no_collate)``, the processors and
  ``flush_buffer``) over the clip in demo_scenario.RUNS, with the detector fakes and a save_mask recorder: every
  detector call (image shape and checksum; SAM's point prompts are left out, they depend on the network's numerics)
  and every save_mask call (frame name, shape, image SHA-256, prompts), in order.
"""
import json
import os
import sys
import tempfile
import types

sys.dont_write_bytecode = True
import make_golden as mg  # noqa: E402  (puts the reference on sys.path, with its shims)

import numpy as np
import torch
from torch.utils.data import DataLoader

import demo_scenario as sc
import detector_masks_scenario as dms


def solve_by_enumeration(pairwise_iou, indicator, total):
    w = [float(pairwise_iou[:, i].sum() * 2) - 1.0 for i in range(total)]
    conflicts = [(i, j) for i in range(total) for j in range(i + 1, total) if indicator[i, j]]
    best_v, best_x = 0.0, 0
    for x in range(1, 1 << total):
        if any((x >> i) & 1 and (x >> j) & 1 for i, j in conflicts):
            continue
        v = sum(w[i] for i in range(total) if (x >> i) & 1)
        if v > best_v + 1e-9:
            best_v, best_x = v, x
    return [bool((best_x >> i) & 1) for i in range(total)]


def main():
    torch.Tensor.cuda = lambda self, *a, **k: self
    for name in ('pycocotools', 'pycocotools.mask', 'supervision'):  # the reference result_utils' imports, unused
        sys.modules.setdefault(name, types.ModuleType(name))
    dms.install_detector_stubs([])
    import deva.inference.consensus_automatic as CA  # pulp is absent: make_golden.golden_consensus' exact enumeration
    CA.use_gurobi = False
    CA.solve_with_pulp = solve_by_enumeration
    from deva.ext import automatic_processor, with_text_processor
    from deva.inference import demo_utils
    from deva.inference.data.simple_video_reader import SimpleVideoReader, no_collate
    for m in (automatic_processor, with_text_processor, demo_utils):
        assert m.__file__.startswith('/root/reference'), m.__file__
    meta, arrays = {'reader': {}, 'ingest': [], 'runs': []}, {}
    with tempfile.TemporaryDirectory() as tmp:
        roots = {'reader': sc.write_reader_folder(os.path.join(tmp, 'reader')),
                 'clip': sc.write_demo_clip(os.path.join(tmp, 'clip'))}
        for name, root in roots.items():
            meta['reader'][name] = sc.read_items(SimpleVideoReader(root), root)
            print(f'  reader {name}: {len(meta["reader"][name])} items')

        for k, (h, w) in enumerate(sc.INGEST_SHAPES):
            for min_side in sc.INGEST_MIN_SIDES:
                out = demo_utils.get_input_frame_for_deva(sc.ingest_frame(h, w, k), min_side)
                key = f'ingest_{k}_{min_side}'
                arrays[key] = out.numpy().astype(np.float32)
                meta['ingest'].append({'key': key, 'hw': [h, w], 'min_side': min_side, 'shape': list(out.shape)})

        sd = mg.param_spec.synthetic_state_dict(seed=1)
        for kind, temporal in sc.RUNS:
            cfg = sc.demo_config(mg.CFG, kind, temporal)
            reader = SimpleVideoReader(roots['clip'])
            cfg['enable_long_term_count_usage'] = bool(cfg['enable_long_term'] and (
                len(reader) / (cfg['max_mid_term_frames'] - cfg['min_mid_term_frames']) * cfg['num_prototypes'])
                >= cfg['max_long_term_elements'])
            net = mg.DEVA(cfg).eval()
            net.load_weights(sd)
            np.random.seed(42)
            deva = mg.DEVAInferenceCore(net, config=cfg)
            args, fakes = sc.detectors(kind, 'cpu')
            saver = sc.SaveRecorder()
            loader = DataLoader(reader, batch_size=None, collate_fn=no_collate, num_workers=0)
            processors = automatic_processor if kind == 'auto' else with_text_processor
            sc.run_demo(processors, demo_utils.flush_buffer, deva, loader, kind, saver, args)
            meta['runs'].append({'kind': kind, 'temporal': temporal, 'detector_calls': sc.calls(fakes, False),
                                 'saves': saver.calls})
            print(f'  run {kind} {temporal}: {len(meta["runs"][-1]["detector_calls"])} detector calls, '
                  f'{len(saver.calls)} saves')
    mg.save('demo.npz', **arrays)
    json.dump(meta, open(os.path.join(mg.HERE, 'demo.json'), 'w'))


if __name__ == '__main__':
    main()
