"""GPU parity of the in-clip consensus (SURVEY 8f-1) against reference-minted fixtures: spatial_alignment and the
established-association average (floating point, through the H100 kernels) and the automatic association's voting
logic (integer: bit-exact ids)."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _scenario(golden_dir):
    spec = importlib.util.spec_from_file_location('consensus_scenario', os.path.join(golden_dir, 'consensus_scenario.py'))
    sc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sc)
    return sc


def _net(cfg, sd):
    from deva.model.network import DEVA
    net = DEVA(cfg).cuda().eval()
    net.load_weights({k: v.cuda() for k, v in sd.items()})
    return net


def _golden(golden_dir):
    g = {k: torch.from_numpy(v) for k, v in np.load(os.path.join(golden_dir, 'consensus.npz')).items()}
    return g, json.load(open(os.path.join(golden_dir, 'consensus.json')))


def test_spatial_alignment_matches_reference(golden_dir, synthetic_sd):
    from deva.inference.consensus_associated import find_consensus_with_established_association, spatial_alignment
    from deva.inference.image_feature_store import ImageFeatureStore
    from deva.utils.tensor_utils import pad_divide_by
    tol = 1e-3
    sc = _scenario(golden_dir)
    g, meta = _golden(golden_dir)
    cfg = meta['config']
    net = _net(cfg, synthetic_sd)
    data = [(im.cuda(), ids.cuda()) for im, ids in sc.frames()]
    store = ImageFeatureStore(net, no_warning=True)
    img0, _ = pad_divide_by(data[0][0], 16)
    img1, _ = pad_divide_by(data[1][0], 16)
    m0, _ = pad_divide_by(torch.stack([data[0][1] == 3, data[0][1] == 5]).float(), 16)
    prob = spatial_alignment(10, img0, m0, 11, img1, net, store, cfg)[0]
    assert tuple(prob.shape) == tuple(g['align_prob'].shape)
    err = float((prob.float().cpu() - g['align_prob']).abs().max())
    print(f'spatial_alignment max |prob - reference| = {err:.3e}')
    assert err < tol, err

    pick = [(0, (3, 5)), (1, (1, 4)), (3, (7, 8))]
    for key, scores in (('established_mask', None), ('established_mask_scored', [0.2, 0.9, 0.5])):
        kti, total = find_consensus_with_established_association(
            [sc.TIMES[i] for i, _ in pick], [data[i][0].clone() for i, _ in pick],
            [torch.stack([data[i][1] == a, data[i][1] == b]).float() for i, (a, b) in pick], net,
            ImageFeatureStore(net, no_warning=True), cfg, scores=scores)
        assert kti == meta['established_keyframe' + ('_scored' if scores else '')]
        err = float((total.float().cpu() - g[key]).abs().max())
        assert err < tol, (key, err)


def _frame_infos(sc, data):
    from deva.inference.frame_utils import FrameInfo
    from deva.inference.object_info import ObjectInfo
    out = []
    for ti, (image, ids), dets in zip(sc.TIMES, data, sc.DETECTIONS):
        infos = [ObjectInfo(sid, category_id=cat, isthing=thing, score=score) for sid, _, cat, thing, score in dets]
        out.append(FrameInfo(image, ids, infos, ti, {}))
    return out


def test_voting_logic_bit_exact(golden_dir, synthetic_sd):
    """Prescribed projections -> matching, exact selection (no ILP solver), meta merging, painting: ids bit-exact."""
    from deva.inference.consensus_automatic import find_consensus_auto_association
    sc = _scenario(golden_dir)
    g, meta = _golden(golden_dir)
    data = [(im.cuda(), ids.cuda()) for im, ids in sc.frames()]
    for keyframe in ('first', 'last', 'middle'):
        kti, mask, infos = find_consensus_auto_association(
            _frame_infos(sc, data), keyframe, network=None, store=None, config=meta['config'],
            align_fn=lambda *a: sc.shifted_alignment(*a[:5]))
        want = meta['auto']['shifted_' + keyframe]
        assert kti == want['keyframe']
        assert [[o.id, o.category_ids, o.scores] for o in infos] == want['segments']
        assert mask.dtype == torch.long and torch.equal(mask.cpu(), g[f'auto_shifted_{keyframe}_mask'])


def test_vote_in_temporary_buffer(golden_dir, synthetic_sd):
    """DEVAInferenceCore.vote_in_temporary_buffer end to end (real projection through the kernels).  The projection
    is floating point, so the id mask may differ from the fp32 reference on a few boundary pixels."""
    from deva.inference.inference_core import DEVAInferenceCore
    sc = _scenario(golden_dir)
    g, meta = _golden(golden_dir)
    net = _net(meta['config'], synthetic_sd)
    core = DEVAInferenceCore(net, meta['config'])
    data = [(im.cuda(), ids.cuda()) for im, ids in sc.frames()]
    for f in _frame_infos(sc, data):
        core.add_to_temporary_buffer(f)
    kti, mask, infos = core.vote_in_temporary_buffer('first')
    want = meta['auto']['real_first']
    assert kti == want['keyframe']
    assert [[o.id, o.category_ids, o.scores] for o in infos] == want['segments']
    ref = g['auto_real_first_mask']
    assert float((mask.cpu() != ref).float().mean()) < 5e-3
    core.clear_buffer()
    assert len(core.image_feature_store) == 0 and core.frame_buffer == []
