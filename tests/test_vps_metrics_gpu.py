"""Device side of the VIPSeg metrics: deva_b200_pano_joint_hist against np.unique over the joint code (both the
shared-memory and the global-atomic histogram), deva_b200_pano_remap against numpy, and merge_stuff / eval_vpq /
eval_stq / eval_vps end to end against the unmodified reference's outputs (tests/golden/vps_metrics.{json,npz}),
including eval_stq called from a process forked after CUDA has been initialised."""
import hashlib
import json
import multiprocessing
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import vps_scenario as vs  # noqa: E402

pytestmark = pytest.mark.gpu
MAX_ID = (1 << 24) - 1


def _frame(rng, h, w, table, n_unknown=3):
    """Blocky id map drawn from the table plus ids that are not in it (up to 2^24 - 1), with per-pixel noise."""
    pool = np.concatenate([table, rng.integers(0, MAX_ID + 1, n_unknown), [MAX_ID]]).astype(np.int64)
    bh, bw = max(1, h // 16), max(1, w // 16)
    blocks = rng.choice(pool, size=((h + bh - 1) // bh, (w + bw - 1) // bw))
    ids = np.repeat(np.repeat(blocks, bh, 0), bw, 1)[:h, :w]
    noise = rng.random((h, w)) < 0.05
    ids[noise] = rng.choice(pool, size=int(noise.sum()))
    return ids


def _rgb(ids):
    return np.stack([(ids >> (8 * i)) & 255 for i in range(3)], -1).astype(np.uint8)


def _table(rng, n):
    return np.unique(rng.integers(0, MAX_ID + 1, 3 * n + 8))[:n].astype(np.int32) if n else np.zeros(0, np.int32)


def _index(ids, table):
    i = np.searchsorted(table, ids)
    ok = (i < len(table)) & (table[np.minimum(i, max(len(table) - 1, 0))] == ids) if len(table) else np.zeros(ids.shape,
                                                                                                            bool)
    return np.where(ok, i, len(table))


@pytest.mark.parametrize('hw', [(1, 1), (7, 13), (720, 1280), (1080, 1920)])
@pytest.mark.parametrize('n_ids', [0, 1, 255, 4096])
def test_joint_hist_matches_numpy(hw, n_ids):
    from deva import _native as nat
    nat.require_device()
    h, w = hw
    rng = np.random.default_rng(h * 7919 + w + n_ids)
    gt_ids, pred_ids = _table(rng, n_ids), _table(rng, max(n_ids - 1, 0) if n_ids > 1 else n_ids)
    g, p = _frame(rng, h, w, gt_ids), _frame(rng, h, w, pred_ids)
    cols = len(pred_ids) + 1
    code = _index(g, gt_ids) * cols + _index(p, pred_ids)
    u, c = np.unique(code, return_counts=True)
    want = np.zeros((len(gt_ids) + 1) * cols, np.int64)
    want[u] = c
    # unaligned frames (byte offset 1) take the byte-load path
    for offset in (0, 1):
        bufs = []
        for a in (_rgb(g), _rgb(p)):
            buf = torch.zeros(a.size + 4, dtype=torch.uint8, device='cuda')
            view = buf[offset:offset + a.size].view(h, w, 3)
            view.copy_(torch.from_numpy(a))
            bufs.append(view)
        hist = torch.full((2, len(gt_ids) + 1, cols), -7, dtype=torch.int32, device='cuda')  # the call initialises it
        nat.pano_joint_hist(bufs[0], bufs[1], torch.from_numpy(gt_ids).cuda(), torch.from_numpy(pred_ids).cuda(), hist[1])
        got = hist[1].cpu().numpy().ravel()
        np.testing.assert_array_equal(got, want)
        assert (hist[0] == -7).all()


@pytest.mark.parametrize('hw', [(1, 1), (37, 53), (720, 1280)])
def test_remap_matches_numpy(hw):
    from deva import _native as nat
    nat.require_device()
    h, w = hw
    rng = np.random.default_rng(h + w)
    table = _table(rng, 200)
    out_ids = np.concatenate([[0], rng.integers(1, MAX_ID + 1, 30)]).astype(np.int32)
    slot = rng.integers(0, len(out_ids), len(table) + 1).astype(np.int32)
    ids = _frame(rng, h, w, table, n_unknown=4)
    s = slot[_index(ids, table)]
    want_out = _rgb(out_ids[s].astype(np.int64))
    want_counts = np.bincount(s.ravel(), minlength=len(out_ids))
    want_unknown = int((_index(ids, table) == len(table)).sum())
    out = torch.empty(h, w, 3, dtype=torch.uint8, device='cuda')
    counts = torch.full((len(out_ids),), -1, dtype=torch.int32, device='cuda')
    unknown = torch.full((1,), -1, dtype=torch.int32, device='cuda')
    nat.pano_remap(torch.from_numpy(_rgb(ids)).cuda(), torch.from_numpy(table).cuda(), torch.from_numpy(slot).cuda(),
                   torch.from_numpy(out_ids).cuda(), out, counts, unknown)
    np.testing.assert_array_equal(out.cpu().numpy(), want_out)
    np.testing.assert_array_equal(counts.cpu().numpy(), want_counts)
    assert int(unknown.item()) == want_unknown


@pytest.fixture(scope='module')
def golden(golden_dir):
    return json.load(open(os.path.join(golden_dir, 'vps_metrics.json'))), np.load(
        os.path.join(golden_dir, 'vps_metrics.npz'))


@pytest.fixture()
def dataset(tmp_path):
    return vs.write_dataset(str(tmp_path))


def test_merge_stuff_matches_reference(golden, dataset, tmp_path):
    from deva.vps_metrics.stuff_merging import merge_stuff
    from deva.vps_metrics.video_pass import read_rgb
    meta, arrays = golden
    out = str(tmp_path / 'merged')
    np.random.seed(meta['merge_seed'])
    merge_stuff(dataset[0], out, isthing={int(k): v for k, v in meta['isthing'].items()})
    assert json.load(open(os.path.join(out, 'pred.json'))) == meta['merged_json']
    for key, digest in meta['merged_sha256'].items():
        px = read_rgb(os.path.join(out, 'pan_pred', key))
        assert hashlib.sha256(px.tobytes()).hexdigest() == digest, key
    for key in arrays.files:
        vid, t = key[len('merged_'):].rsplit('_', 1)
        np.testing.assert_array_equal(read_rgb(os.path.join(out, 'pan_pred', vid, f'{int(t):08d}.png')), arrays[key])
    # in place, as evaluation/eval_with_detections.py calls it
    np.random.seed(meta['merge_seed'])
    merge_stuff(dataset[0], dataset[0], isthing={int(k): v for k, v in meta['isthing'].items()})
    assert json.load(open(os.path.join(dataset[0], 'pred.json'))) == meta['merged_json']


def _files(submit):
    return {n: open(os.path.join(submit, n)).read() for n in sorted(os.listdir(submit)) if n.endswith('.txt')}


@pytest.mark.parametrize('entry', ['eval_vpq', 'eval_stq', 'eval_vps'])
def test_metrics_match_reference(golden, dataset, entry):
    import deva.vps_metrics as vm
    from deva.vps_metrics.eval_stq_vipseg import eval_stq
    from deva.vps_metrics.eval_vpq_vipseg import eval_vpq
    meta, _ = golden
    submit = dataset[0]
    {'eval_vpq': lambda: eval_vpq(*dataset, num_processes=4), 'eval_stq': lambda: eval_stq(*dataset),
     'eval_vps': lambda: vm.eval_vps(*dataset)}[entry]()
    files = _files(submit)
    want = {k: v for k, v in meta['files'].items() if (k == 'stq.txt') == (entry == 'eval_stq') or entry == 'eval_vps'}
    assert files == want


@pytest.mark.parametrize('kind', ['png', 'json', 'unlisted'])
def test_prediction_key_error_on_device(golden, dataset, kind):
    """'unlisted' lands in the kernel's not-in-table bucket; the id is then named from the PNG."""
    from deva.vps_metrics.eval_vpq_vipseg import eval_vpq
    meta, _ = golden
    vs.break_prediction(dataset[0], kind)
    with pytest.raises(KeyError) as e:
        eval_vpq(*dataset)
    assert e.value.args[0] == meta['errors'][kind]


def test_eval_stq_in_forked_child(golden, dataset):
    from deva.vps_metrics.eval_stq_vipseg import eval_stq
    meta, _ = golden
    torch.zeros(1, device='cuda')  # CUDA is initialised in this process, as in the driver
    assert torch.cuda.is_initialized()
    child = multiprocessing.get_context('fork').Process(target=eval_stq, args=dataset)
    child.start()
    child.join()
    assert child.exitcode == 0
    assert _files(dataset[0]) == {'stq.txt': meta['files']['stq.txt']}
