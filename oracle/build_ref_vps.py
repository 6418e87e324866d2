"""Recipe: stage the UNMODIFIED reference's VIPSeg metric modules (``deva/vps_metrics``) under ``oracle/_ref/`` next to
what build_ref.py stages (build container only).

    python oracle/build_ref.py && python oracle/build_ref_vps.py   # both run by __graft_entry__.build()

Run after build_ref.py, which recreates ``oracle/_ref/`` from scratch.  The files are copied byte for byte (git-ignored,
like the rest of ``oracle/_ref/``) and listed with their hashes in ``oracle/_ref/MANIFEST_vps_metrics.json``.  What uses
them: ``tools/bench_vps_metrics.py``, which times the reference's stuff merging, VPQ and STQ against this package's on
the same host.  Where the reference is absent (the GPU box), the staged copy that travelled there is kept as is.
"""
import hashlib
import json
import os
import shutil
import sys

from build_ref import DST, SRC

PART = 'deva/vps_metrics'


def build() -> bool:
    src, dst = os.path.join(SRC, PART), os.path.join(DST, PART)
    if not os.path.isdir(src):
        print(f'[oracle/_ref] {src} not present (GPU box): keeping the staged copy as is', file=sys.stderr)
        return os.path.isdir(dst)
    if os.path.isdir(dst):
        shutil.rmtree(dst)
    shutil.copytree(src, dst, ignore=shutil.ignore_patterns('__pycache__', '*.pyc'))
    manifest = {os.path.relpath(os.path.join(root, f), DST): hashlib.sha256(open(os.path.join(root, f), 'rb').read())
                .hexdigest()[:16] for root, _, files in os.walk(dst) for f in sorted(files)}
    json.dump({'source': SRC, 'files': manifest}, open(os.path.join(DST, 'MANIFEST_vps_metrics.json'), 'w'), indent=0)
    print(f'[oracle/_ref] staged {len(manifest)} files of {PART} from {SRC}')
    return True


if __name__ == '__main__':
    sys.exit(0 if build() else 1)
