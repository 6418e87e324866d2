"""CPU: multi-scale / flip evaluation's host logic (member spec, mapping -> lut) and the self-consistency of the
fixture minted from the unmodified reference by tests/golden/make_multiscale_golden.py."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fixture(golden_dir):
    return (np.load(os.path.join(golden_dir, 'multiscale_vos.npz')),
            json.load(open(os.path.join(golden_dir, 'multiscale_vos.json'))))


def _merge_loop(total, mapping):
    """scripts/merge_multi_scale.py::process_vid on one frame's summed scores."""
    result = np.argmax(total.astype(np.float32), axis=0)
    idx = np.zeros_like(result, dtype=np.uint8)
    for l, i in mapping.items():
        idx[result == i] = l
    return idx


def test_module_imports_without_gpu():
    code = ("import sys, torch\n"
            "import deva.inference.multi_scale as m\n"
            "assert m.__file__.startswith(sys.argv[1]), m.__file__\n"
            "from deva.inference.frame_io import prob_to_scores, scores_to_ids\n")
    pkg = os.path.join(ROOT, 'tracking-anything-with-deva_b200')
    env = dict(os.environ, PYTHONPATH=pkg, CUDA_VISIBLE_DEVICES='')
    out = subprocess.run([sys.executable, '-c', code, pkg], env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


def test_member_spec_is_validated():
    from deva.inference.multi_scale import validate_members
    assert validate_members([(240, False), (None, True), [480, True]]) == [(240, False), (None, True), (480, True)]
    for bad in ([], [(240,)], [240], [(0, False)], [(-1, False)], [(240.0, False)], [(True, False)], [(240, 1)],
                [('240', False)]):
        with pytest.raises(ValueError):
            validate_members(bad)


def test_mapping_lut_follows_the_merge_loop():
    from deva.inference.frame_io import mapping_lut
    rng = np.random.default_rng(0)
    c = 7
    mappings = [{}, {1: 1, 2: 2}, {7: 1, 3: 2, 200: 3}, {5: 2, 9: 2},  # 9 overwrites 5 on channel 2
                {4: 0, 6: 3}, {8: 1, 11: 9, 12: -1},  # channel 0 mapped; channels outside [0, c) ignored
                {300: 1, 2: 1, 17: 4}]
    for mapping in mappings:
        lut = np.array(mapping_lut(mapping, c))
        for _ in range(3):
            argmax_map = rng.integers(0, c, (9, 11))
            onehot = (argmax_map[None] == np.arange(c)[:, None, None]).astype(np.int32)
            small = {l: i for l, i in mapping.items() if l < 256}  # numpy refuses to store ids above 255 in uint8
            if len(small) == len(mapping):
                assert np.array_equal(lut[argmax_map].astype(np.uint8), _merge_loop(onehot, mapping)), mapping
        last = {}
        for l, i in mapping.items():
            last[i] = l
        assert lut.tolist() == [last.get(k, 0) for k in range(c)], mapping


def test_fixture_is_self_consistent(golden_dir):
    g, meta = _fixture(golden_dir)
    members = [tuple(m) for m in meta['members']]
    assert members == [(s, f) for s in (240, 360, 480) for f in (False, True)]
    lat = g['scores_lattice'].astype(np.int64)  # [members, T, K+1, h, w]
    total = g['sum_lattice']
    assert lat.shape[0] == len(members) and lat.shape[1:] == total.shape
    assert np.array_equal(lat.sum(0), total)
    T, H, W = g['ids'].shape
    assert [H, W] == meta['shape'] and T == len(meta['frames'])
    mapping = {int(k): v for k, v in meta['mapping'].items()}
    assert sorted(mapping) == sorted(meta['labels'])
    step = meta['lattice']
    for t in range(T):
        assert np.array_equal(_merge_loop(total[t], mapping), g['ids'][t, ::step, ::step]), t
    decided = np.unpackbits(g['decided'])[:T * H * W].reshape(T, H, W).astype(bool)
    assert decided[0].mean() > 0.5
