import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'tracking-anything-with-deva_b200')
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on the H100 box with -m gpu)')


@pytest.fixture(scope='session')
def golden_dir():
    return GOLDEN


@pytest.fixture(scope='session')
def synthetic_sd():
    """Synthetic checkpoint seed 1 (the one tests/golden/make_golden.py used)."""
    from deva.model.param_spec import synthetic_state_dict
    return synthetic_state_dict(seed=1)
