"""PNG files decoded on the device (csrc/png_decode.cu, deva/utils/png_decode.py): Pillow's array or exception for
every case of tests/golden/png_decode_cases.py, with the device's statuses equal to oracle/png_decode.py's eligibility
and acceptance; mixed batches with fallbacks among them; repeatable results; and the post-processing passes with
png_decoder='device' reproducing tests/golden/unsup_davis17.* and tests/golden/vps_metrics.*."""
import io
import json
import multiprocessing
import os
import re
import sys

import numpy as np
import pytest
import torch
from PIL import Image

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
sys.path.insert(0, GOLDEN)
import png_decode_cases as pdc  # noqa: E402
import vps_scenario as vs  # noqa: E402

from oracle import png_decode as od  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def cases():
    return pdc.cases(large=True)


def _pillow(data):
    try:
        return np.asarray(Image.open(io.BytesIO(data)))
    except Exception as e:  # noqa: BLE001
        return e


def _message(e):
    return re.sub(r' at 0x[0-9a-f]+>', '>', str(e))  # Pillow names an in-memory file by its object's address


def _assert_same(got, want, case):
    if isinstance(want, BaseException):
        assert type(got) is type(want) and _message(got) == _message(want), (case, got, want)
    else:
        assert isinstance(got, torch.Tensor) and got.is_cuda, (case, got)
        got = got.cpu().numpy()
        assert got.dtype == want.dtype and got.shape == want.shape, (case, got.dtype, got.shape, want.shape)
        np.testing.assert_array_equal(got, want, err_msg=case)


def test_statuses_match_oracle(cases):
    """One batch of the whole matrix: a status of 0 exactly where the oracle accepts, and the oracle's array there."""
    from deva.utils import png_decode
    files = [(d, png_decode.parse(d)) for _, d in cases]
    results = png_decode.decode_batch(files)
    for (case, data), (status, t) in zip(cases, results):
        info = od.eligible(data)
        assert (status is None) == (info is None), case
        if info is not None:
            assert (status == 0) == od.accepts(info), (case, status)
        if status == 0:
            np.testing.assert_array_equal(t.cpu().numpy(), _pillow(data), err_msg=case)


def test_decode_matches_pillow(cases, tmp_path):
    """decode_results over bytes and paths (a missing path among them): Pillow's array or exception for every file."""
    from deva.utils.png_decode import decode_results
    sources = [d for _, d in cases]
    for got, (case, data) in zip(decode_results(sources), cases):
        _assert_same(got, _pillow(data), case)
    paths = []
    for k, (case, data) in enumerate(cases[:200]):
        p = tmp_path / f'{k}.png'
        p.write_bytes(data)
        paths.append(str(p))
    paths.insert(7, str(tmp_path / 'missing.png'))
    for got, p in zip(decode_results(paths), paths):
        try:
            want = np.asarray(Image.open(p))
        except Exception as e:  # noqa: BLE001
            want = e
        _assert_same(got, want, p)


def test_mixed_batches_with_fallbacks_and_a_small_budget(cases):
    """Mixed sizes and modes with refused and ineligible files among them, split over several batches."""
    from deva.utils.png_decode import decode_results
    rng = np.random.default_rng(7)
    picked = [cases[int(i)] for i in rng.permutation(len(cases))[:300]]
    for budget in (1 << 16, 1 << 22):
        for got, (case, data) in zip(decode_results([d for _, d in picked], budget=budget), picked):
            _assert_same(got, _pillow(data), case)


def test_public_api_raises_pillows_error(cases):
    from deva.utils.png_decode import decode_png, decode_pngs
    c = dict(cases)
    t = decode_png(c['fixture-png_decode_davis_bmx-trees_00000.png'])
    np.testing.assert_array_equal(t.cpu().numpy(), _pillow(c['fixture-png_decode_davis_bmx-trees_00000.png']))
    with pytest.raises(OSError, match='broken data stream'):
        decode_pngs([c['pil-RGB-l6-45x67'], c['quirk-bad-adler']])


def test_repeated_decodes_are_identical(cases):
    from deva.utils.png_decode import decode_results
    big = [d for case, d in cases if case.startswith(('pil-RGB-ellipse', 'fixture', 'dev-RGB-ellipse'))]
    first = [t.cpu() for t in decode_results(big)]
    for _ in range(2):
        for a, b in zip(first, decode_results(big)):
            assert torch.equal(a, b.cpu())


# ---------------------------------------------------------------------------------------------- post-processing
@pytest.fixture()
def statuses(monkeypatch):
    """The device statuses of every file the passes send to png_decode.decode_batch (None: not eligible)."""
    from deva.utils import png_decode
    seen, decode_batch = [], png_decode.decode_batch

    def recording(files, device=None):
        out = decode_batch(files, device)
        seen.extend(s for s, _ in out)
        return out
    monkeypatch.setattr(png_decode, 'decode_batch', recording)
    return seen


def _pngs(*dirs):
    return sum(f.endswith('.png') for d in dirs for _, _, fs in os.walk(d) for f in fs)


def _assert_device_decoded(statuses, n=None):
    """The device decoded the files (status 0) and refused none; with n, exactly n files, all on the device."""
    decoded = sum(s == 0 for s in statuses)
    assert decoded > 0 and all(s in (0, None) for s in statuses), statuses
    if n is not None:
        assert decoded == len(statuses) == n, (decoded, len(statuses), n)


def test_limit_max_id_with_device_decoder(tmp_path, statuses):
    import unsup_davis_scenario as us
    from deva.inference.postprocess_unsup_davis17 import limit_max_id
    meta = json.load(open(os.path.join(GOLDEN, 'unsup_davis17.json')))
    arrays = np.load(os.path.join(GOLDEN, 'unsup_davis17.npz'))
    palette = bytes.fromhex(meta['palette'])
    for case in us.CASES:
        root = tmp_path / case
        root.mkdir()
        error, files = us.run_case(
            lambda src, dst, m: limit_max_id(src, dst, m, palette=palette, png_decoder='device'), str(root), case)
        us.assert_matches(meta, arrays, case, error, files)
    _assert_device_decoded(statuses)  # the scenario's unreadable and unsupported files go to read_frame


def test_limit_max_id_reads_the_environment(tmp_path, monkeypatch, statuses):
    import unsup_davis_scenario as us
    from deva.inference.postprocess_unsup_davis17 import limit_max_id
    meta = json.load(open(os.path.join(GOLDEN, 'unsup_davis17.json')))
    arrays = np.load(os.path.join(GOLDEN, 'unsup_davis17.npz'))
    palette = bytes.fromhex(meta['palette'])
    monkeypatch.setenv('DEVA_B200_PNG_DECODER', 'device')
    case = next(iter(us.CASES))
    error, files = us.run_case(lambda src, dst, m: limit_max_id(src, dst, m, palette=palette), str(tmp_path), case)
    us.assert_matches(meta, arrays, case, error, files)
    _assert_device_decoded(statuses)


@pytest.fixture(scope='module')
def vps_golden():
    return json.load(open(os.path.join(GOLDEN, 'vps_metrics.json'))), np.load(os.path.join(GOLDEN, 'vps_metrics.npz'))


def _files(submit):
    return {n: open(os.path.join(submit, n)).read() for n in sorted(os.listdir(submit)) if n.endswith('.txt')}


def test_merge_stuff_with_device_decoder(vps_golden, tmp_path, statuses):
    import hashlib
    from deva.vps_metrics.stuff_merging import merge_stuff
    from deva.vps_metrics.video_pass import read_rgb
    meta, arrays = vps_golden
    dataset = vs.write_dataset(str(tmp_path))
    out = str(tmp_path / 'merged')
    np.random.seed(meta['merge_seed'])
    merge_stuff(dataset[0], out, isthing={int(k): v for k, v in meta['isthing'].items()}, png_decoder='device')
    assert json.load(open(os.path.join(out, 'pred.json'))) == meta['merged_json']
    for key, digest in meta['merged_sha256'].items():
        assert hashlib.sha256(read_rgb(os.path.join(out, 'pan_pred', key)).tobytes()).hexdigest() == digest, key
    _assert_device_decoded(statuses, _pngs(os.path.join(dataset[0], 'pan_pred')))


@pytest.mark.parametrize('entry', ['eval_vpq', 'eval_stq', 'eval_vps', 'env'])
def test_metrics_with_device_decoder(vps_golden, tmp_path, monkeypatch, statuses, entry):
    import deva.vps_metrics as vm
    from deva.vps_metrics.eval_stq_vipseg import eval_stq
    from deva.vps_metrics.eval_vpq_vipseg import eval_vpq
    meta, _ = vps_golden
    dataset = vs.write_dataset(str(tmp_path))
    n = _pngs(os.path.join(dataset[0], 'pan_pred'), dataset[1])
    if entry == 'env':
        monkeypatch.setenv('DEVA_B200_PNG_DECODER', 'device')
        vm.eval_vps(*dataset)
    else:
        {'eval_vpq': lambda: eval_vpq(*dataset, num_processes=4, png_decoder='device'),
         'eval_stq': lambda: eval_stq(*dataset, png_decoder='device'),
         'eval_vps': lambda: vm.eval_vps(*dataset, png_decoder='device')}[entry]()
    want = {k: v for k, v in meta['files'].items() if (k == 'stq.txt') == (entry == 'eval_stq') or
            entry in ('eval_vps', 'env')}
    assert _files(dataset[0]) == want
    _assert_device_decoded(statuses, n)


@pytest.mark.parametrize('kind', ['png', 'json', 'unlisted'])
def test_prediction_key_error_with_device_decoder(vps_golden, tmp_path, kind):
    from deva.vps_metrics.eval_vpq_vipseg import eval_vpq
    meta, _ = vps_golden
    dataset = vs.write_dataset(str(tmp_path))
    vs.break_prediction(dataset[0], kind)
    with pytest.raises(KeyError) as e:
        eval_vpq(*dataset, png_decoder='device')
    assert e.value.args[0] == meta['errors'][kind]


def _forked_stq(dataset):
    from deva.vps_metrics.eval_stq_vipseg import eval_stq
    eval_stq(*dataset, png_decoder='device')


def test_eval_stq_in_forked_child_with_device_decoder(vps_golden, tmp_path):
    meta, _ = vps_golden
    dataset = vs.write_dataset(str(tmp_path))
    torch.zeros(1, device='cuda')
    assert torch.cuda.is_initialized()
    child = multiprocessing.get_context('fork').Process(target=_forked_stq, args=(dataset,))
    child.start()
    child.join()
    assert child.exitcode == 0
    assert _files(dataset[0]) == {'stq.txt': meta['files']['stq.txt']}
