"""The wide top-k fixture (tests/golden/topk_wide, minted from the reference at top_k 50 and 100) and the wide entry
points' declarations.  No GPU."""
import json
import os
import re

import numpy as np
import torch

from oracle import memory_math as mm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
WIDE = ('deva_b200_sim_topk_wide_workspace_bytes', 'deva_b200_sim_topk_wide', 'deva_b200_merge_lists_wide',
        'deva_b200_readout_sparse_wide_workspace_bytes', 'deva_b200_readout_sparse_wide',
        'deva_b200_readout_sparse_scatter_wide')


def _fixture():
    g = dict(np.load(os.path.join(GOLDEN, 'topk_wide.npz')))
    meta = json.load(open(os.path.join(GOLDEN, 'topk_wide.json')))
    return g, meta


def test_fixture_is_self_consistent():
    g, meta = _fixture()
    assert meta['top_ks'] == [50, 100]
    for k in meta['top_ks']:
        cfg, sizes = meta['configs'][str(k)], meta['sizes'][str(k)]
        assert cfg['top_k'] == k and len(sizes) == 16
        n, q = g[f'k{k}_read_sim'].shape
        assert n >= k, 'the first read must already hold top_k slots'
        for t in range(16):
            p = g[f'k{k}_prob_{t:02d}']
            assert p.shape == ((3 if t < 6 else 4), 40, 48)
            assert np.abs(p.sum(0) - 1).max() < 1e-5 and p.min() >= 0
            ids = g[f'k{k}_ids_{t:02d}']
            assert ids.shape == (160, 192)
            assert set(np.unique(ids).tolist()) <= ({0, 1, 2} if t < 6 else {0, 1, 2, 7})
            conf = np.unpackbits(g[f'k{k}_confident_{t:02d}'])
            assert conf.size == 160 * 192
        assert sizes[0] == {'0': [120, 0]} and sizes[-1] == {'0': [600, 256], '1': [1080, 0]}


def test_topk_softmax_reproduces_the_fixture_reads():
    g, meta = _fixture()
    for k in meta['top_ks']:
        sim = torch.from_numpy(g[f'k{k}_read_sim']).double()
        aff = torch.from_numpy(g[f'k{k}_read_aff']).double()
        got = mm.dense_affinity(sim, k)
        assert int((aff > 0).sum(0).min()) == k
        assert float((got - aff).abs().max()) < 1e-6


def _header():
    text = open(os.path.join(ROOT, 'include', 'deva_b200.h')).read()
    return re.sub(r'/\*.*?\*/', ' ', text, flags=re.S)


def test_wide_symbols_are_declared_and_exported():
    from deva import _native
    header = _header()
    for name in WIDE:
        assert re.search(r'DEVA_B200_API\s+\w+\s*\**\s*' + name + r'\s*\(', header), name
        assert name in _native.EXPORTS
    so = os.path.join(ROOT, 'tracking-anything-with-deva_b200', 'csrc', 'libdeva_b200.so')
    if os.path.exists(so):   # built: the symbols resolve
        _native.lib()
        assert all(hasattr(_native.lib(), name) for name in WIDE)


def test_list_pitch():
    from deva import _native
    assert [_native.list_pitch(k) for k in (1, 30, 32, 33, 64, 65, 1000)] == [32, 32, 32, 64, 64, 96, 1024]
