"""VIPSeg VPQ / STQ / stuff merging from per-frame joint histograms (oracle/vps_metrics.py, numpy) against the unmodified
reference's outputs in tests/golden/vps_metrics.{json,npz} (minted by make_vps_golden.py on vps_scenario's dataset):
every stat, the JSON and the text files equal, floats bit for bit.  No GPU."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

from oracle import vps_metrics as ov
from deva.vps_metrics import scoring

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import vps_scenario as vs  # noqa: E402


@pytest.fixture(scope='module')
def golden(golden_dir):
    return json.load(open(os.path.join(golden_dir, 'vps_metrics.json'))), np.load(
        os.path.join(golden_dir, 'vps_metrics.npz'))


@pytest.fixture(scope='module')
def dataset(tmp_path_factory):
    return vs.write_dataset(str(tmp_path_factory.mktemp('vps')))


def stat_json(stat):
    return {str(k): [float(v.iou).hex(), int(v.tp), int(v.fp), int(v.fn)] for k, v in stat.items()}


def test_vpq_and_stq_match_reference(golden, dataset):
    meta, _ = golden
    vpq_stats, stq_metric, categories_list = ov.evaluate(*dataset)
    for n in scoring.NFRAMES:
        ours = {k: v for k, v in stat_json(vpq_stats[n]).items() if v != ['0x0.0p+0', 0, 0, 0]}
        ref = {k: v for k, v in meta['vpq_stats'][str(n)]['total'].items() if v != ['0x0.0p+0', 0, 0, 0]}
        assert ours == ref, n
    r = stq_metric.result()
    for key in ('STQ', 'AQ', 'IoU'):
        assert float(r[key]).hex() == meta['stq'][key], key
    assert [float(v).hex() for v in r['AQ_per_seq']] == meta['stq']['AQ_per_seq']
    assert [float(v).hex() for v in r['IoU_per_seq']] == meta['stq']['IoU_per_seq']
    assert [int(v) for v in r['Length_per_seq']] == meta['stq']['Length_per_seq']
    # the text files, byte for byte
    categories = {el['id']: el for el in categories_list}
    vpqs = []
    for n in scoring.NFRAMES:
        results = scoring.vpq_results(vpq_stats[n], categories)
        assert scoring.vpq_text(results) == meta['files'][f'vpq-{n}.txt'], n
        vpqs.append((100 * results['All']['pq'], 100 * results['Things']['pq'], 100 * results['Stuff']['pq']))
    assert scoring.vpq_simple_text(vpqs) == meta['files']['vpq-simple.txt']
    assert scoring.stq_text(r) == meta['files']['stq.txt']


def test_stuff_merging_matches_reference(golden, dataset):
    meta, arrays = golden
    isthing = {int(k): v for k, v in meta['isthing'].items()}
    assert isthing == vs.ISTHING
    np.random.seed(meta['merge_seed'])
    out_json, images = ov.merge_stuff(dataset[0], isthing)
    assert json.loads(json.dumps(out_json)) == meta['merged_json']
    assert {k: hashlib.sha256(v.tobytes()).hexdigest() for k, v in images.items()} == meta['merged_sha256']
    for key in arrays.files:  # merged_<video>_<t>
        vid, t = key[len('merged_'):].rsplit('_', 1)
        np.testing.assert_array_equal(images[f'{vid}/{int(t):08d}.png'], arrays[key])


def test_fixture_is_self_consistent(golden, dataset):
    meta, arrays = golden
    # per-video stats add up to the totals (PQStat.__iadd__, video by video)
    for n, entry in meta['vpq_stats'].items():
        total = {}
        for video in entry['per_video']:
            for k, (iou, tp, fp, fn) in video.items():
                t = total.setdefault(k, [0.0, 0, 0, 0])
                total[k] = [t[0] + float.fromhex(iou), t[1] + tp, t[2] + fp, t[3] + fn]
        assert {k: [v[0].hex()] + v[1:] for k, v in total.items()} == entry['total'], n
    # the scenario's features are present: exactly-0.5 IoU, ids >= 2^16, a random draw in merging, the 720p video
    submit, truth, gt_path = dataset
    gt = json.load(open(gt_path))
    assert any(el['id'] >= 1 << 16 for v in gt['annotations'] for f in v['annotations'] for el in f['segments_info'])
    assert any(el['iscrowd'] for v in gt['annotations'] for f in v['annotations'] for el in f['segments_info'])
    merged_ids = {el['id'] for v in meta['merged_json']['annotations'] for f in v['annotations']
                  for el in f['segments_info']}
    pred = json.load(open(os.path.join(submit, 'pred.json')))
    pred_ids = {el['id'] for v in pred['annotations'] for f in v['annotations'] for el in f['segments_info']}
    assert merged_ids - pred_ids, 'no id was drawn at random'
    assert [len(f) for f in (vs.make_video('v_one'),)] == [1]
    assert sum(k.startswith('v_720p/') for k in meta['merged_sha256']) == vs.VIDEOS['v_720p'][0]
    assert len(arrays.files) == sum(t for name, (t, *_rest) in vs.VIDEOS.items() if name != 'v_720p')
    g, p = ov.decode(np.array(ov.video_pass.read_rgb(os.path.join(truth, 'v_small', '00000000.png')))), ov.decode(
        ov.video_pass.read_rgb(os.path.join(submit, 'pan_pred', 'v_small', '00000000.png')))
    inter, union = ((g == 4242) & (p == 4243)).sum(), ((g == 4242) | (p == 4243)).sum()
    assert inter * 2 == union


@pytest.mark.parametrize('kind', ['png', 'json', 'unlisted'])
def test_prediction_key_errors(golden, dataset, tmp_path, kind):
    import shutil
    meta, _ = golden
    submit, truth, gt_path = dataset
    broken = str(tmp_path / 'submit')
    shutil.copytree(submit, broken)
    vs.break_prediction(broken, kind)
    with pytest.raises(KeyError) as e:
        ov.evaluate(broken, truth, gt_path)
    assert e.value.args[0] == meta['errors'][kind]
