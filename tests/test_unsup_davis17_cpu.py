"""Unsupervised DAVIS 2017 post-processing without a GPU: the numpy restatement (oracle/unsup_davis17.py) against the
unmodified reference's outputs in tests/golden/unsup_davis17.{json,npz} (minted by make_unsup_davis_golden.py on
unsup_davis_scenario's inputs), the fixture's own consistency and coverage, and an import that leaves CUDA alone."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import unsup_davis17 as ou

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import unsup_davis_scenario as us  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def golden(golden_dir):
    return json.load(open(os.path.join(golden_dir, 'unsup_davis17.json'))), np.load(
        os.path.join(golden_dir, 'unsup_davis17.npz'))


@pytest.mark.parametrize('case', list(us.CASES))
def test_oracle_matches_reference(golden, tmp_path, case):
    meta, arrays = golden
    palette = bytes.fromhex(meta['palette'])
    error, files = us.run_case(lambda src, dst, m: ou.limit_max_id(src, dst, m, palette), str(tmp_path), case)
    us.assert_matches(meta, arrays, case, error, files)


def test_fixture_is_self_consistent(golden):
    meta, arrays = golden
    palette = bytes.fromhex(meta['palette'])
    assert len(palette) == 768 and us.sha(palette) == meta['palette_sha256']
    assert set(meta['cases']) == set(us.CASES)
    for case, entry in meta['cases'].items():
        for k, (mode, pal, digest, shape) in entry['files'].items():
            assert mode == 'P' and pal == meta['palette_sha256'], (case, k)
            if f'{case}/{k}' in arrays:
                px = arrays[f'{case}/{k}']
                assert us.sha(px.tobytes()) == digest and list(px.shape) == shape
    cases = meta['cases']
    # max = 0: every mask all zero; a negative max: the assert, nothing written
    assert all(not arrays[f'max0/{k}'].any() for k in cases['max0']['files'])
    assert cases['negative'] == {'error': ['AssertionError', ''], 'files': {}}
    # the overflow: the earlier video written, the failing one and the later one not
    assert cases['overflow']['error'][0] == 'OverflowError'
    assert {k.split(os.sep)[0] for k in cases['overflow']['files']} == {'a'}
    # in place writes what a separate output directory gets; the empty video writes nothing
    assert cases['in_place']['files'] == cases['max20']['files']
    assert not any(k.startswith('zzz_empty') for k in cases['max20']['files'])
    assert [shape for shape in (v[3] for v in cases['hd']['files'].values())] == [[1080, 1920]] * 2


def test_scenario_covers_the_rules(golden):
    meta, arrays = golden
    base = us.DATASETS['base']
    labels = {vid: [us.frame_labels(v, t) for t in range(v[1])] for vid, v in base.items()}
    # labels >= 2^16, and an area tie that R-major order breaks the other way from the saver's colour order
    assert max(int(f.max()) for f in labels['car']) >= 1 << 16
    assert any((f == us.R1).sum() == (f == us.R2).sum() > 0 for f in labels['car'])
    assert us.R2 > us.R1 and (us.R2 & 255) * 65536 + (us.R2 >> 16) < (us.R1 & 255) * 65536 + (us.R1 >> 16)
    # bear: three labels in every frame fill 20 entries after 7 frames, so each label's index comes from a later
    # duplicate, and the label first seen after the break becomes 0
    bear = [arrays[f'max20/bear/{t:05d}.png'] for t in range(9)]
    assert all(len(np.unique(f[f != 0])) == 3 for f in labels['bear'][:7])
    got = np.unique(bear[0][4:]).tolist()
    assert len(got) == 3 and min(got) >= 16 and max(got) == 20, got  # frames 5 and 6 hold the last positions
    assert (labels['bear'][8][0:3, 0:5] == 9).all() and not bear[8][0:3, 0:5].any()
    # all-zero input frames stay zero, and RGBA / L / P / RGB inputs are all present
    assert not labels['dog'][0].any() and not arrays['max20/dog/00000.png'].any()
    assert {v[0] for v in base.values()} == {'P', 'L', 'RGB', 'RGBA'}
    assert 'dog/00005.PNG' in meta['cases']['max20']['files']


def test_import_leaves_cuda_uninitialised():
    code = ('import sys, torch; sys.path[:0] = [{!r}, {!r}]; '
            'import deva.inference.postprocess_unsup_davis17 as m; import deva.vps_metrics.video_pass; '
            'assert m.__file__.startswith({!r}), m.__file__; '
            'assert not torch.cuda.is_initialized(); print("ok")').format(
                ROOT, os.path.join(ROOT, 'tracking-anything-with-deva_b200'),
                os.path.join(ROOT, 'tracking-anything-with-deva_b200'))
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip() == 'ok', out.stderr
