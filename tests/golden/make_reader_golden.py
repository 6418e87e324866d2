"""Mint the dataset-reader fixture from the UNMODIFIED reference readers on the CPU (build container only).

    python tests/golden/make_reader_golden.py

Builds reader_scenario.clip_files(), writes the clips to a temporary directory, and runs every reader_scenario.RUNS
entry through the reference's deva/inference/data/video_reader.py and detection_video_reader.py (pycocotools, which
video_reader imports for a path no run takes, and pulp, which the package's __init__ imports, are stubbed as
make_golden.py and make_ingest_golden.py do).  For every item it stores
``default_collate([reader[i]])`` - its structure and dtypes in readers.json, its small tensors in readers.npz, and the
float frames (and resized soft masks) as the sha256 of their bytes - or the type and message of the error the item or
its collate raises.  readers.npz also holds the bytes of every synthetic clip file, so the tests read the files the
fixture was made from; the real bmx-trees and vipseg files are read from their own files in tests/golden.
"""
import json
import os
import sys
import tempfile
import types

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, '/root/reference')
coco = types.ModuleType('pycocotools')
coco.mask = types.ModuleType('pycocotools.mask')
sys.modules['pycocotools'], sys.modules['pycocotools.mask'] = coco, coco.mask
sys.modules['pulp'] = types.ModuleType('pulp')  # the reference package's __init__ reaches it; the readers do not

import numpy as np  # noqa: E402
from torch.utils.data import default_collate  # noqa: E402

import reader_scenario as sc  # noqa: E402
from deva.inference.data.detection_video_reader import DetectionVideoReader  # noqa: E402
from deva.inference.data.video_reader import VideoReader  # noqa: E402

assert VideoReader.__module__ == 'deva.inference.data.video_reader' and '/root/reference' in sys.modules[
    'deva.inference.data.video_reader'].__file__


def main():
    files = sc.clip_files()
    arrays = {f'file/{rel}': np.frombuffer(data, np.uint8) for rel, data in files.items()}
    files.update(sc.real_files())
    meta = {'runs': {}}
    with tempfile.TemporaryDirectory() as root:
        sc.materialise(files, root)
        classes = {'VideoReader': VideoReader, 'DetectionVideoReader': DetectionVideoReader}
        for run in sc.RUNS:
            name = run[0]
            try:
                reader = sc.make_reader(classes, run, root)
            except Exception as e:  # noqa: BLE001
                meta['runs'][name] = {'init_error': sc.error_record(e, root)}
                print(name, 'init error', type(e).__name__)
                continue
            items = []
            for i in range(len(reader)):
                try:
                    item = default_collate([reader[i]])
                    items.append(sc.record(item, root, f'run/{name}/{i}', arrays))
                except Exception as e:  # noqa: BLE001
                    items.append(sc.error_record(e, root))
            meta['runs'][name] = {'len': len(reader), 'items': items}
            print(name, len(reader), [('E:' + it['error']) if 'error' in it else 'ok' for it in items])
    np.savez_compressed(os.path.join(HERE, 'readers.npz'), **arrays)
    json.dump(meta, open(os.path.join(HERE, 'readers.json'), 'w'), indent=0)
    print('wrote readers.npz', len(arrays), 'arrays')


if __name__ == '__main__':
    main()
