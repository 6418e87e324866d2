"""Recipe: stage the UNMODIFIED reference's SAM automatic mask generator as DEVA vendors it
(``deva/ext/SAM/__init__.py``, ``deva/ext/SAM/automatic_mask_generator.py``) under ``oracle/_ref/``, next to what
build_ref.py and build_ref_ext.py stage (build container only).

    python oracle/build_ref.py && python oracle/build_ref_sam.py   # both run by __graft_entry__.build()

Run after build_ref.py, which recreates ``oracle/_ref/`` from scratch.  The files are copied byte for byte (git-ignored,
like the rest of ``oracle/_ref/``) and listed with their hashes in ``oracle/_ref/MANIFEST_sam.json``.  What uses them:
oracle/sam_masks.py, which loads the generator by path over the stand-in ``segment_anything`` of oracle/sam_stub.py,
for tests/golden/make_sam_masks_golden.py, tests/test_sam_masks_gpu.py (the reference generator run live, and
``deva.ext.SAM`` for ``get_sam_model(..., mask_generator='reference')``) and tools/bench_sam_masks.py.  Where the
reference is absent (the GPU box), the staged copy that travelled there is kept as is.
"""
import hashlib
import json
import os
import shutil
import sys

from build_ref import DST, SRC

FILES = ('deva/ext/SAM/__init__.py', 'deva/ext/SAM/automatic_mask_generator.py')


def build() -> bool:
    if not all(os.path.isfile(os.path.join(SRC, f)) for f in FILES):
        print(f'[oracle/_ref] {SRC}/deva/ext/SAM not present (GPU box): keeping the staged copy as is', file=sys.stderr)
        return all(os.path.isfile(os.path.join(DST, f)) for f in FILES)
    manifest = {}
    for f in FILES:
        dst = os.path.join(DST, f)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copy2(os.path.join(SRC, f), dst)
        manifest[f] = hashlib.sha256(open(dst, 'rb').read()).hexdigest()[:16]
    json.dump({'source': SRC, 'files': manifest}, open(os.path.join(DST, 'MANIFEST_sam.json'), 'w'), indent=0)
    print(f'[oracle/_ref] staged {len(manifest)} files of deva/ext/SAM from {SRC}')
    return True


if __name__ == '__main__':
    sys.exit(0 if build() else 1)
