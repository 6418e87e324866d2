"""The device JPEG decoder (deva/utils/jpeg_decode.py, csrc/jpeg_decode.cu) against Pillow: every eligible file's array
equal to ``np.asarray(Image.open(f))`` from 1x1 to 4K, Pillow's exception for every file Pillow refuses, results in
order for mixed batches, and a nonzero status for every corrupt stream whose array would differ."""
import io
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tracking-anything-with-deva_b200'))
import jpeg_decode_cases as jdc  # noqa: E402

pytestmark = pytest.mark.gpu


def pillow(data):
    from PIL import Image
    try:
        return np.asarray(Image.open(io.BytesIO(data)))
    except Exception as e:  # noqa: BLE001
        return e


@pytest.fixture(scope='module')
def valid():
    return jdc.valid_cases() + jdc.valid_cases(large=True)


def same_message(a, b):
    """Pillow's messages name the BytesIO object they read; its address differs between two opens."""
    def strip(e):
        return re.sub(r' at 0x[0-9a-f]+', '', str(e))
    return strip(a) == strip(b)


def device_statuses(files):
    from deva.utils import jpeg_decode as jd
    return jd.decode_batch([(f, jd.parse(f)) for f in files])


def test_device_arrays_equal_pillow(valid):
    from deva.utils import jpeg_decode as jd
    files = [f for _, f in valid]
    declined = []
    for (cid, f), (st, t) in zip(valid, device_statuses(files)):
        assert st is not None, cid  # every valid case is eligible
        if st != 0:
            declined.append((cid, st))
            continue
        assert np.array_equal(t.cpu().numpy(), pillow(f)), cid
    # only quality-1 content and custom tables may leave the IDCT's agreed range
    assert all(cid.startswith(('noise-37x53-q1-', 'overlay-37x53-q1-', 'gradient-37x53-q1-', 'qtables', 'saturated'))
               for cid, _ in declined), declined
    assert len(declined) <= len(valid) // 20, declined
    for cid, f in valid[:40]:
        assert np.array_equal(jd.decode_jpeg(f).cpu().numpy(), pillow(f)), cid


def test_mixed_batch_in_order(valid):
    from deva.utils import jpeg_decode as jd
    small = [f for cid, f in valid if '1080' not in cid and '2160' not in cid][::7]
    mixed = []
    bad = [f for _, f in jdc.ineligible()]
    corrupt = [f for _, f in jdc.mutants(small, 20, seed=3)]
    for k in range(max(len(small), len(bad), len(corrupt))):
        for group in (small, bad, corrupt):
            if k < len(group):
                mixed.append(group[k])
    out = jd.decode_results(mixed)
    assert len(out) == len(mixed)
    for f, r in zip(mixed, out):
        want = pillow(f)
        if isinstance(want, Exception):
            assert type(r) is type(want) and same_message(r, want)
        else:
            assert isinstance(r, torch.Tensor) and r.is_cuda and np.array_equal(r.cpu().numpy(), want)


def test_repeated_decodes_identical(valid):
    files = [f for cid, f in valid if '1080' in cid][:2] + [f for _, f in valid[:30]]
    first = [t.clone() if t is not None else None for _, t in device_statuses(files)]
    for _ in range(3):
        for a, (_, b) in zip(first, device_statuses(files)):
            assert (a is None) == (b is None) and (a is None or torch.equal(a, b))


def test_mutants_status_zero_only_with_pillows_array(valid):
    from deva.utils import jpeg_decode as jd
    base = [f for cid, f in valid if cid.startswith(('overlay-120x200', 'restart', 'encode_jpeg', 'jpeg_decode'))]
    files = [f for _, f in jdc.mutants(base, 400, seed=11)]
    accepted = 0
    for f, (st, t) in zip(files, device_statuses(files)):
        if st == 0:
            accepted += 1
            assert np.array_equal(t.cpu().numpy(), pillow(f))
        else:
            assert st is None or st > 0
    print(f'mutants accepted by the device: {accepted}/{len(files)}')


def test_extreme_coefficients_equal_pillow_or_refused():
    cases = jdc.extreme()
    refused = 0
    for (cid, f), (st, t) in zip(cases, device_statuses([f for _, f in cases])):
        if st == 0:
            assert np.array_equal(t.cpu().numpy(), pillow(f)), cid
        else:
            refused += 1
    assert 0 < refused < len(cases)


def test_async_decode_does_not_synchronise(valid):
    from deva.utils import jpeg_decode as jd
    f = next(f for cid, f in valid if cid == 'overlay-480x854-q75')
    hd = jd.parse(f)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        frame, status, keep = jd.decode_async(hd)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert int(status.item()) == 0
    assert np.array_equal(frame.cpu().numpy(), pillow(f))
