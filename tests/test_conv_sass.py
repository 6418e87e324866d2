"""The convolution kernel's machine code keeps its wgmma pipeline asynchronous and its accumulators in registers.

ptxas silently serializes wgmma (every instruction waits for the previous group to drain) when one sits in a divergent
path, and spills to local memory when the accumulator does not fit the register budget; both cost most of the
tensor-core rate without changing any result, so only the SASS shows them.  No GPU needed.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'tracking-anything-with-deva_b200', 'csrc', 'libdeva_b200.so')


def _cuobjdump():
    found = shutil.which('cuobjdump')
    if found:
        return found
    for home in (os.environ.get('CUDA_HOME'), os.environ.get('CUDA_PATH'), '/usr/local/cuda'):
        if home and os.path.isfile(os.path.join(home, 'bin', 'cuobjdump')):
            return os.path.join(home, 'bin', 'cuobjdump')
    return None


def _conv_kernels():
    """{mangled name: SASS text} of every conv_kernel instantiation in the built library."""
    tool = _cuobjdump()
    if tool is None or not os.path.isfile(LIB):
        pytest.skip('needs the built library and cuobjdump')
    sass = subprocess.run([tool, '-sass', LIB], check=True, capture_output=True, text=True).stdout
    funcs, name = {}, None
    for line in sass.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            name = m.group(1) if 'conv_kernel' in m.group(1) else None
            if name:
                funcs[name] = []
        elif name:
            funcs[name].append(line)
    return {k: '\n'.join(v) for k, v in funcs.items()}


def test_conv_kernels_pipeline_wgmma_without_spills():
    funcs = _conv_kernels()
    assert len(funcs) == 9, sorted(funcs)  # {64, 128, 192, 256} x {plain, head} + the 192-wide gate epilogue
    for name, text in funcs.items():
        spills = re.findall(r'\b(?:STL|LDL)\b', text)
        in_flight = len(re.findall(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b', text))
        drains = len(re.findall(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b', text))
        assert not spills, f'{name}: {len(spills)} local-memory accesses (register spills)'
        assert in_flight >= 1, f'{name}: no wgmma group is ever left in flight (serialized pipeline)'
        assert drains <= 1, f'{name}: {drains} full drains of the wgmma pipeline (expected one, before the epilogue)'
