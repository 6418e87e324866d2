"""The JPEG decoder's host side and its CPU restatements (deva/utils/jpeg_decode.py, oracle/jpeg_decode.py and the host
build of csrc/jpeg_decode.cuh) against Pillow: the oracle's array equals ``np.asarray(Image.open(f))`` on every
eligible file, the eligibility rule refuses what Pillow must decide, and the device's parallel algorithm, run serially,
equals the sequential decode at every subsequence size and gives status 0 only with Pillow's array."""
import io
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tracking-anything-with-deva_b200'))
import jpeg_decode_cases as jdc  # noqa: E402
from deva.utils import jpeg_decode as jd  # noqa: E402
from oracle import jpeg_decode as oj  # noqa: E402

ORACLE_BYTES = 60000  # the oracle's bit-by-bit Huffman decode is slow; larger files go through the host build only


def pillow(data):
    from PIL import Image
    try:
        return np.asarray(Image.open(io.BytesIO(data)))
    except Exception as e:  # noqa: BLE001
        return e


@pytest.fixture(scope='module')
def valid():
    return jdc.valid_cases()


@pytest.fixture(scope='module')
def host(tmp_path_factory):
    nvcc = '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(nvcc):
        pytest.skip('nvcc is not installed')
    exe = str(tmp_path_factory.mktemp('jpeg') / 'jpeg_decode_host')
    csrc = os.path.join(ROOT, 'tracking-anything-with-deva_b200', 'csrc')
    subprocess.run([nvcc, '-x', 'cu', '-O2', '-std=c++17', '-I', csrc,
                    os.path.join(ROOT, 'tests', 'native', 'jpeg_decode_host.cu'), '-o', exe],
                   check=True, capture_output=True)

    def run(headers, sub_bytes):
        """-> [(sequential status, parallel status, rounds, agree, array or None)] per Header."""
        inp = b''
        for hd in headers:
            inp += struct.pack('<6i', hd.h, hd.w, hd.hy, hd.vy, sub_bytes, len(hd.intervals))
            inp += b''.join(struct.pack('<4q', *iv) for iv in hd.intervals)
            inp += hd.tables.astype('<i4').tobytes() + struct.pack('<q', len(hd.scan)) + hd.scan.tobytes()
        out = subprocess.run([exe], input=inp, capture_output=True, check=True).stdout
        res, p = [], 0
        for hd in headers:
            s1, s2, rounds, same = struct.unpack_from('<4i', out, p)
            p += 16
            img = None
            if s2 == 0:
                img = np.frombuffer(out, np.uint8, hd.nbytes, p).reshape(hd.shape)
                p += hd.nbytes
            res.append((s1, s2, rounds, same, img))
        assert p == len(out)
        return res
    return run


def test_oracle_matches_pillow(valid):
    checked = 0
    for cid, f in valid:
        if len(f) > ORACLE_BYTES:
            continue
        st, img = oj.decode(f)
        assert st == 0, (cid, st)
        assert np.array_equal(img, pillow(f)), cid
        checked += 1
    assert checked > 250


def test_every_valid_case_is_eligible(valid):
    for cid, f in valid + jdc.valid_cases(large=True):
        hd = jd.parse(f)
        assert hd is not None, cid
        assert hd.shape == pillow(f).shape, cid


@pytest.mark.parametrize('cid', [c for c, _ in jdc.ineligible()])
def test_ineligible_files_go_to_pillow(cid):
    f = dict(jdc.ineligible())[cid]
    assert jd.parse(f) is None
    assert oj.decode(f) is None


def test_extreme_coefficients_equal_pillow_or_refused(host):
    cases = jdc.extreme()
    statuses = []
    for (cid, f), (s1, s2, _, same, img) in zip(cases, host([jd.parse(f) for _, f in cases], 128)):
        st, ref = oj.decode(f)
        assert s1 == s2 == st and same, cid
        if st == 0:
            assert np.array_equal(img, pillow(f)) and np.array_equal(ref, img), cid
        statuses.append(st)
    # the range check must both accept extreme files that Pillow agrees with and refuse some
    assert statuses.count(0) and statuses.count(oj.RANGE)


@pytest.mark.parametrize('sub_bytes', [1, 7, 32, 128])
def test_parallel_algorithm_equals_sequential_small(host, valid, sub_bytes):
    small = [(c, f) for c, f in valid if len(f) < 20000 or sub_bytes >= 32]
    res = host([jd.parse(f) for _, f in small], sub_bytes)
    for (cid, f), (s1, s2, rounds, same, img) in zip(small, res):
        assert s1 == s2 == 0 and same, (cid, s1, s2)
        assert np.array_equal(img, pillow(f)), cid
    print(f'subsequence {sub_bytes} B: at most {max(r[2] for r in res)} synchronisation rounds')


@pytest.mark.parametrize('sub_bytes', [128, 1024])
def test_parallel_algorithm_equals_sequential_large(host, sub_bytes):
    large = jdc.valid_cases(large=True)
    res = host([jd.parse(f) for _, f in large], sub_bytes)
    rounds = []
    for (cid, f), (s1, s2, r, same, img) in zip(large, res):
        assert s1 == s2 == 0 and same, (cid, s1, s2)
        assert np.array_equal(img, pillow(f)), cid
        rounds.append((cid, r))
    print(f'subsequence {sub_bytes} B: synchronisation rounds {rounds}')


def test_mutants_status_zero_only_with_pillows_array(host, valid):
    base = [f for cid, f in valid if cid.startswith(('overlay-120x200', 'restart', 'encode_jpeg-overlay-37', 'qtables',
                                                     'overlay-37x53'))]
    files = [f for _, f in jdc.mutants(base, 3000, seed=7)]
    eligible = [(f, jd.parse(f)) for f in files]
    eligible = [(f, hd) for f, hd in eligible if hd is not None]
    accepted = 0
    for sub in (16, 128):
        for (f, hd), (s1, s2, _, same, img) in zip(eligible, host([hd for _, hd in eligible], sub)):
            assert same
            if s2 == 0:
                accepted += 1
                assert np.array_equal(img, pillow(f))
    for f, _ in eligible[:150]:
        st, img = oj.decode(f)
        (s1, _, _, _, ref), = host([jd.parse(f)], 128)
        assert (st == 0) == (s1 == 0) and (st != 0 or np.array_equal(img, ref))
    assert 0 < accepted < 2 * len(eligible)


def test_resolve_decoder(monkeypatch):
    monkeypatch.delenv(jd.ENV, raising=False)
    assert jd.resolve_decoder() == 'pil'
    monkeypatch.setenv(jd.ENV, 'device')
    assert jd.resolve_decoder() == 'device'
    assert jd.resolve_decoder('pil') == 'pil'
    with pytest.raises(ValueError):
        jd.resolve_decoder('nvjpeg')


def test_import_leaves_cuda_uninitialised():
    code = ('import sys; sys.path[:0] = [{!r}, {!r}]; import torch; from deva.utils import jpeg_decode; '
            'from oracle import jpeg_decode as o; print(torch.cuda.is_initialized())').format(
        ROOT, os.path.join(ROOT, 'tracking-anything-with-deva_b200'))
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, check=True).stdout
    assert out.strip() == 'False'
