"""Mint the unsupervised DAVIS 2017 post-processing fixture from the UNMODIFIED reference on the CPU (build container
only).

    python tests/golden/make_unsup_davis_golden.py

Runs the reference's ``limit_max_id`` (deva/inference/postprocess_unsup_davis17.py, with its default DAVIS palette) on
every case of unsup_davis_scenario.CASES and records what it raised and every file of the output tree afterwards: mode,
palette hash and pixels.  Writes unsup_davis17.json (the palette bytes as hex, per case the error and per file the mode,
the palette's sha256 and the pixels' sha256) and unsup_davis17.npz (the pixels of every file under 100 000 pixels).
"""
import json
import os
import sys
import tempfile

sys.dont_write_bytecode = True
import make_golden as mg  # noqa: E402  (puts the reference first on sys.path, with its shims)

import numpy as np  # noqa: E402

import unsup_davis_scenario as us  # noqa: E402
from deva.inference import postprocess_unsup_davis17 as ref  # noqa: E402
from deva.utils.palette import davis_palette  # noqa: E402

assert ref.__file__.startswith('/root/reference'), ref.__file__


def main():
    meta = {'palette': bytes(davis_palette).hex(), 'palette_sha256': us.sha(bytes(davis_palette)), 'cases': {}}
    arrays = {}
    for case in us.CASES:
        with tempfile.TemporaryDirectory() as root:
            error, files = us.run_case(ref.limit_max_id, root, case)
        meta['cases'][case] = {'error': error, 'files': {k: [mode, pal, us.sha(px.tobytes()), list(px.shape)]
                                                         for k, (mode, pal, px) in sorted(files.items())}}
        for k, (_, _, px) in files.items():
            if px.size < 100000:
                arrays[f'{case}/{k}'] = px
        print(case, error, len(files), 'files')
    mg.save('unsup_davis17.npz', **arrays)
    json.dump(meta, open(os.path.join(mg.HERE, 'unsup_davis17.json'), 'w'), indent=0)


if __name__ == '__main__':
    main()
