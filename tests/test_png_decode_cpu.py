"""The PNG decoder without a GPU: oracle/png_decode.py against Pillow over tests/golden/png_decode_cases.py and a
hypothesis sweep, the host eligibility rule of deva/utils/png_decode.py against the oracle's, the allowlisted chunks
against Pillow, and a host build of csrc/inflate.cuh against zlib on valid streams, malformed ones and a few thousand
seeded mutants."""
import io
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
sys.path.insert(0, GOLDEN)
import png_decode_cases as pdc  # noqa: E402

from oracle import png_decode as od  # noqa: E402

CASES = pdc.cases(large=False)


def pillow(data):
    """('array', array) or ('error', type, message) of np.asarray(Image.open(data))."""
    try:
        return ('array', np.asarray(Image.open(io.BytesIO(data))))
    except Exception as e:  # noqa: BLE001
        return ('error', type(e), str(e))


def check_oracle(data):
    info = od.eligible(data)
    if info is None or not od.accepts(info):
        return False
    kind, *got = pillow(data)
    assert kind == 'array', got
    want = od.decode(info)
    assert got[0].dtype == want.dtype and got[0].shape == want.shape
    np.testing.assert_array_equal(got[0], want)
    return True


@pytest.mark.parametrize('case', [c for c, _ in CASES])
def test_oracle_matches_pillow(case):
    data = dict(CASES)[case]
    accepted = check_oracle(data)
    if not case.startswith(('quirk', 'hdr', 'blk', 'sym', 'dist', 'stream', 'file', 'mode')):
        assert accepted, case  # every well-formed file of the matrix is decoded on the device


def test_malformed_files_are_refused():
    """Every malformed case is either ineligible or refused by the device's acceptance rule, and Pillow's result for
    it is what the module's docstring says (the quirks)."""
    for case, data in pdc.malformed():
        info = od.eligible(data)
        assert info is None or not od.accepts(info), case
    quirks = dict(pdc.malformed())
    assert pillow(quirks['quirk-bad-idat-crc'])[0] == 'array'
    assert pillow(quirks['quirk-trailing-bytes'])[0] == 'array'
    assert pillow(quirks['quirk-extra-inflated'])[0] == 'array'
    assert pillow(quirks['quirk-bad-adler'])[1:] == (OSError, 'broken data stream when reading image file')
    assert pillow(quirks['quirk-filter-5'])[1:] == (OSError, 'unrecognized data stream contents when reading image '
                                                             'file')
    short = pillow(quirks['quirk-stream-ends-early'])
    assert short[0] == 'error' or not short[1][-1].any()


def test_host_rule_matches_oracle():
    from deva.utils import png_decode
    for case, data in CASES:
        hd, info = png_decode.parse(data), od.eligible(data)
        assert (hd is None) == (info is None), case
        if hd is not None:
            assert (hd.h, hd.w, hd.colour_type, hd.bits, hd.mode, hd.stream(data)) == info, case


@pytest.mark.parametrize('mode,bits', [('L', 8), ('L', 2), ('RGB', 8), ('RGBA', 8), ('P', 4)])
def test_allowlisted_chunks_leave_pillow_unchanged(mode, bits):
    img = pdc.image('ellipse', mode, 21, 33, levels=1 << bits if mode in ('L', 'P') else 256)
    plain = pillow(pdc.build(img, mode, bits))[1]
    for kind, data in pdc.ANCILLARY:
        if kind == b'tRNS' and mode == 'RGBA':
            continue
        f = pdc.build(img, mode, bits, before=[(kind, pdc.ancillary_data(kind, data, mode))])
        assert od.eligible(f) is not None, kind
        got = pillow(f)[1]
        assert got.dtype == plain.dtype and got.shape == plain.shape, kind
        np.testing.assert_array_equal(got, plain)
    f = pdc.build(img, mode, bits, after=[(b'tEXt', b'k\x00v'), (b'tIME', pdc.ANCILLARY[-1][1])])
    np.testing.assert_array_equal(pillow(f)[1], plain)


@settings(max_examples=150, deadline=None)
@given(st.sampled_from([('L', 2), ('L', 4), ('L', 8), ('P', 1), ('P', 2), ('P', 4), ('P', 8), ('RGB', 8),
                        ('RGBA', 8)]), st.integers(1, 24), st.integers(1, 40), st.integers(0, 2 ** 32 - 1),
       st.sampled_from([0, 1, 6, 9]), st.sampled_from([zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY,
                                                       zlib.Z_RLE, zlib.Z_FIXED]), st.sampled_from([9, 11, 15]))
def test_oracle_matches_pillow_on_random_images(fmt, h, w, seed, level, strategy, wbits):
    mode, bits = fmt
    rng = np.random.default_rng(seed)
    img = pdc.image(['ellipse', 'noise', 'gradient'][seed % 3], mode, h, w, seed, pdc.levels_of(mode, bits))
    filters = [int(v) for v in rng.integers(0, 5, h)]
    f = pdc.build(img, mode, bits, filters, level, strategy, wbits, split=[int(v) for v in rng.integers(0, 9, seed % 4)])
    assert check_oracle(f)


# ---------------------------------------------------------------------------------------------- host inflate
KTRAILING = 11


@pytest.fixture(scope='module')
def inflate_host(tmp_path_factory):
    nvcc = '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(nvcc):
        pytest.skip('nvcc is not installed')
    exe = str(tmp_path_factory.mktemp('inflate') / 'inflate_host')
    csrc = os.path.join(ROOT, 'tracking-anything-with-deva_b200', 'csrc')
    subprocess.run([nvcc, '-x', 'cu', '-O2', '-std=c++17', '-I', csrc, os.path.join(ROOT, 'tests', 'native',
                                                                                    'inflate_host.cu'), '-o', exe],
                   check=True, capture_output=True)

    def run(items):
        """items: [(stream, expected length)] -> [(status, bytes or None)]."""
        inp = b''.join(struct.pack('<I', len(s)) + s + struct.pack('<Q', n) for s, n in items)
        out = subprocess.run([exe], input=inp, capture_output=True, check=True).stdout
        res, p = [], 0
        for _ in items:
            status, n = struct.unpack_from('<iQ', out, p)
            p += 12
            res.append((status, out[p:p + n] if status == 0 else None))
            p += n if status == 0 else 0
        assert p == len(out)
        return res
    return run


def zlib_result(stream):
    """zlib's reading of a stream: (inflated bytes, trailing bytes) or None when zlib refuses it or it ends early."""
    d = zlib.decompressobj()
    try:
        out = d.decompress(stream)
    except zlib.error:
        return None
    return (out, d.unused_data) if d.eof else None


def check_against_zlib(run, streams, expect_valid=None):
    """For every stream zlib reads whole, the core gives zlib's bytes (or kTrailing when bytes follow the stream);
    for every other stream, a nonzero status."""
    items, wants = [], []
    for s in streams:
        z = zlib_result(s)
        wants.append(z)
        items.append((s, len(z[0]) if z else 1000))
    for s, z, (status, got) in zip(streams, wants, run(items)):
        if z is None:
            assert status != 0, s[:16]
        elif z[1]:
            assert status == KTRAILING, status
        else:
            assert status == 0 and got == z[0], status
        if expect_valid is not None:
            assert (z is not None and not z[1]) == expect_valid


def test_host_inflate_matches_zlib_on_valid_streams(inflate_host):
    streams = [od.eligible(d)[5] for _, d in CASES if od.eligible(d) is not None]
    streams = [s for s in streams if zlib_result(s) and not zlib_result(s)[1]]
    raw = bytes(np.random.default_rng(1).integers(0, 3, 300000, dtype=np.uint8)) + b'xyz' * 40000
    for strategy in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED):
        for level in (0, 1, 5, 9):
            for wbits in (9, 12, 15):
                co = zlib.compressobj(level, zlib.DEFLATED, wbits, 8, strategy)
                streams.append(co.compress(raw) + co.flush())
    streams.append(zlib.compress(b''))
    check_against_zlib(inflate_host, streams, expect_valid=True)


def test_host_inflate_refuses_malformed_streams(inflate_host):
    streams = []
    for case, data in pdc.malformed():
        info = od.eligible(data)
        if info is not None:
            streams.append(info[5])
    check_against_zlib(inflate_host, streams)
    # and with the length the PNG asks for: every malformed eligible file is refused (filter types are the unfilter
    # pass's to check)
    items = []
    for case, data in pdc.malformed():
        info = od.eligible(data)
        if info is not None and not case.startswith('quirk-filter'):
            h, w, _, bits, mode, s = info
            items.append((s, h * ((w * od.CHANNELS[mode] * bits + 7) // 8 + 1)))
    assert all(status != 0 for status, _ in inflate_host(items))


def test_host_inflate_on_mutants(inflate_host):
    """Seeded bit flips and truncations of streams from every writer: the core agrees with zlib on each."""
    rng = np.random.default_rng(2024)
    bases = [od.eligible(d)[5] for c, d in CASES if c.startswith(('pil-', 'cv-', 'dev-', 'zlib-')) and
             len(od.eligible(d)[5]) < 20000][::3]
    streams = []
    for k in range(3000):
        s = bytearray(bases[k % len(bases)])
        if k % 4 == 3:
            streams.append(bytes(s[:int(rng.integers(0, len(s)))]))
            continue
        for _ in range(1 + k % 3):
            i = int(rng.integers(0, len(s)))
            s[i] ^= 1 << int(rng.integers(0, 8))
        streams.append(bytes(s))
    check_against_zlib(inflate_host, streams)


def test_import_does_not_initialise_cuda():
    code = ('import torch, deva.utils.png_decode, deva.utils.png_pipeline; '
            'assert not torch.cuda.is_initialized()')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, 'tracking-anything-with-deva_b200')]))
    subprocess.run([sys.executable, '-c', code], check=True, env=env)


def test_resolve_decoder(monkeypatch):
    from deva.utils.png_decode import resolve_decoder
    monkeypatch.delenv('DEVA_B200_PNG_DECODER', raising=False)
    assert resolve_decoder() == 'pil'
    monkeypatch.setenv('DEVA_B200_PNG_DECODER', 'device')
    assert resolve_decoder() == 'device' and resolve_decoder('pil') == 'pil'
    with pytest.raises(ValueError, match='png_decoder'):
        resolve_decoder('gpu')


def test_batches_respect_the_budget():
    from deva.utils.png_decode import Header, batches
    hd = Header(100, 100, 2, 8, 'RGB', ())
    assert batches([hd] * 10, budget=2 * 30000 * 3 + 300) == [(0, 3), (3, 6), (6, 9), (9, 10)]
    assert batches([hd, None, hd], budget=60100) == [(0, 2), (2, 3)]  # an ineligible file costs nothing
