"""Recipe: stage the UNMODIFIED reference's detector-mask modules (``deva/ext/__init__.py``, ``automatic_sam.py``,
``grounding_dino.py``) under ``oracle/_ref/`` next to what build_ref.py stages (build container only).

    python oracle/build_ref.py && python oracle/build_ref_ext.py   # both run by __graft_entry__.build()

Run after build_ref.py, which recreates ``oracle/_ref/`` from scratch.  The files are copied byte for byte (git-ignored,
like the rest of ``oracle/_ref/``) and listed with their hashes in ``oracle/_ref/MANIFEST_ext.json``.  What uses them:
``tools/bench_detector_masks.py``, which loads them by path, with stub detector modules, and times the reference's
``auto_segment`` / ``segment_with_text`` against this package's on the same GPU.  Where the reference is absent (the GPU
box), the staged copy that travelled there is kept as is.
"""
import hashlib
import json
import os
import shutil
import sys

from build_ref import DST, SRC

FILES = ('deva/ext/__init__.py', 'deva/ext/automatic_sam.py', 'deva/ext/grounding_dino.py')


def build() -> bool:
    if not all(os.path.isfile(os.path.join(SRC, f)) for f in FILES):
        print(f'[oracle/_ref] {SRC}/deva/ext not present (GPU box): keeping the staged copy as is', file=sys.stderr)
        return all(os.path.isfile(os.path.join(DST, f)) for f in FILES)
    manifest = {}
    for f in FILES:
        dst = os.path.join(DST, f)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copy2(os.path.join(SRC, f), dst)
        manifest[f] = hashlib.sha256(open(dst, 'rb').read()).hexdigest()[:16]
    json.dump({'source': SRC, 'files': manifest}, open(os.path.join(DST, 'MANIFEST_ext.json'), 'w'), indent=0)
    print(f'[oracle/_ref] staged {len(manifest)} files of deva/ext from {SRC}')
    return True


if __name__ == '__main__':
    sys.exit(0 if build() else 1)
