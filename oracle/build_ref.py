"""Recipe: stage the UNMODIFIED reference's propagation path under ``oracle/_ref/`` (build container only).

    python oracle/build_ref.py          # also run by __graft_entry__.build() when /root/reference exists

The reference (hkchengrex/Tracking-Anything-with-DEVA @ 404a112) is pure Python, so "building" it is staging the
files its propagation path imports - ``deva/inference``, ``deva/model``, ``deva/utils`` - byte for byte where they lie
under /root/reference, into ``oracle/_ref/`` (git-ignored, NOT gpurun-ignored: it travels to the GPU box like a
built ``.so``; no reference source enters the repository history).  ``pip install /root/reference`` is not possible
here (the build backend ``hatchling`` is absent and there is no index); outcome recorded in DESIGN.md.

What uses it (test infrastructure / reported baselines only, never the product path):
  * ``bench.py --impl reference``      - the reference's own ``DEVAInferenceCore.step`` on the host cores;
  * ``bench.py``'s ``torch_gpu_baseline`` - the same unmodified code on the same H100 (fp32, fp32 without TF32, --amp).
``oracle/ref_loader.py`` imports it in a process that never imports the product's ``deva`` package.
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.environ.get('DEVA_REFERENCE_ROOT', '/root/reference')
DST = os.path.join(HERE, '_ref')
PARTS = ('deva/__init__.py', 'deva/inference', 'deva/model', 'deva/utils')


def build() -> bool:
    if not os.path.isdir(os.path.join(SRC, 'deva')):
        print(f'[oracle/_ref] {SRC} not present (GPU box): keeping the staged copy as is', file=sys.stderr)
        return os.path.isdir(os.path.join(DST, 'deva'))
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    os.makedirs(DST)
    manifest = {}
    for part in PARTS:
        src = os.path.join(SRC, part)
        dst = os.path.join(DST, part)
        if os.path.isdir(src):
            shutil.copytree(src, dst, ignore=shutil.ignore_patterns('__pycache__', '*.pyc', '*.txt', 'data'))
        else:
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            shutil.copy2(src, dst)
    for root, _, files in os.walk(DST):
        for f in sorted(files):
            path = os.path.join(root, f)
            manifest[os.path.relpath(path, DST)] = hashlib.sha256(open(path, 'rb').read()).hexdigest()[:16]
    json.dump({'source': SRC, 'files': manifest}, open(os.path.join(DST, 'MANIFEST.json'), 'w'), indent=0)
    print(f'[oracle/_ref] staged {len(manifest)} files from {SRC}')
    return True


if __name__ == '__main__':
    sys.exit(0 if build() else 1)
