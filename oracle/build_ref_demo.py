"""Recipe: stage the UNMODIFIED reference's demo processors (``deva/ext/automatic_processor.py``,
``with_text_processor.py``) and the ``deva/dataset`` modules the reference's ``demo_utils`` imports (``__init__.py``,
``utils.py``) under ``oracle/_ref/``, next to what build_ref.py and build_ref_ext.py stage (build container only).

    python oracle/build_ref.py && python oracle/build_ref_ext.py && python oracle/build_ref_demo.py
    # all three run by __graft_entry__.build()

Run after build_ref.py, which recreates ``oracle/_ref/`` from scratch.  The files are copied byte for byte (git-ignored,
like the rest of ``oracle/_ref/``) and listed with their hashes in ``oracle/_ref/MANIFEST_demo.json``.  What uses them:
tests/test_demo_gpu.py, which runs the unmodified processors over a demo clip with this package first on the path, and
tools/bench_demo.py, which also times the reference's own ``demo_utils`` ingest (staged by build_ref.py with the rest
of ``deva/inference``).  Where the reference is absent (the GPU box), the staged copy that travelled there is kept as
is.
"""
import hashlib
import json
import os
import shutil
import sys

from build_ref import DST, SRC

FILES = ('deva/ext/automatic_processor.py', 'deva/ext/with_text_processor.py', 'deva/dataset/__init__.py',
         'deva/dataset/utils.py')


def build() -> bool:
    if not all(os.path.isfile(os.path.join(SRC, f)) for f in FILES):
        print(f'[oracle/_ref] {SRC} demo processors not present (GPU box): keeping the staged copy as is',
              file=sys.stderr)
        return all(os.path.isfile(os.path.join(DST, f)) for f in FILES)
    manifest = {}
    for f in FILES:
        dst = os.path.join(DST, f)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copy2(os.path.join(SRC, f), dst)
        manifest[f] = hashlib.sha256(open(dst, 'rb').read()).hexdigest()[:16]
    json.dump({'source': SRC, 'files': manifest}, open(os.path.join(DST, 'MANIFEST_demo.json'), 'w'), indent=0)
    print(f'[oracle/_ref] staged {len(manifest)} files of the demos (deva/ext processors, deva/dataset) from {SRC}')
    return True


if __name__ == '__main__':
    sys.exit(0 if build() else 1)
