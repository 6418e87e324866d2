"""GPU: the detector-mask kernels against torch on the device, and the auto_segment / segment_with_text drop-ins against
the fixture minted from the unmodified reference."""
import importlib.util
import json
import os
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# |area - torch's sum| <= AREA_RTOL * torch's sum + AREA_ATOL: both are fp32 sums of the same values in different orders
AREA_RTOL, AREA_ATOL = 2e-5, 1e-3


@pytest.fixture(scope='module')
def nat():
    from deva import _native
    _native.require_device()
    return _native


@pytest.fixture(scope='module')
def sc(golden_dir):
    spec = importlib.util.spec_from_file_location('detector_masks_scenario',
                                                  os.path.join(golden_dir, 'detector_masks_scenario.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def random_masks(n, h, w, seed, dup=True):
    """bool [n, h, w] on the device: blobs of varied size plus noise; mask 1 repeats mask 0 when n > 2."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    if n == 0:
        return torch.zeros((0, h, w), dtype=torch.bool, device='cuda')
    coarse = torch.rand((n, 1, max(1, h // 16), max(1, w // 16)), generator=g, device='cuda')
    blobs = F.interpolate(coarse, (h, w), mode='bilinear')[:, 0]
    thr = torch.rand((n, 1, 1), generator=g, device='cuda')
    m = (blobs > thr) ^ (torch.rand((n, h, w), generator=g, device='cuda') < 0.02)
    if dup and n > 2:
        m[1] = m[0]
    return m.contiguous()


def torch_resized(masks, out_h, out_w):
    if masks.shape[0] == 0:  # F.interpolate rejects an empty stack
        return torch.zeros((0, out_h, out_w), device=masks.device)
    return F.interpolate(masks.float()[None], (out_h, out_w), mode='bilinear')[0]


SIZES = [((1, 1), (1, 1)), ((37, 53), (20, 29)), ((64, 80), (64, 80)), ((1080, 1920), (480, 853)),
         ((240, 427), (480, 854)), ((96, 128), (48, 64)), ((5, 3), (11, 7))]
CASES = [(n, s) for n in (0, 1, 2, 31, 33) for s in SIZES] + \
        [(257, s) for s in SIZES if s[0][0] < 1000] + [(1500, ((37, 53), (20, 29))), (1500, ((96, 128), (48, 64)))]


@pytest.mark.parametrize('n,size', CASES)
@pytest.mark.parametrize('dtype', [torch.bool, torch.uint8])
def test_mask_stats(nat, n, size, dtype):
    (h, w), (oh, ow) = size
    masks = random_masks(n, h, w, seed=n * 31 + h).to(dtype)
    area = torch.full((n,), -1.0, device='cuda')
    covered = torch.full((n,), -1, dtype=torch.int32, device='cuda')
    nat.mask_stats(masks, oh, ow, area, covered)
    v = torch_resized(masks, oh, ow)
    assert torch.equal(covered.long(), (v > 0.5).flatten(1).sum(1))
    ref = v.flatten(1).sum(1)
    assert bool(((area - ref).abs() <= AREA_RTOL * ref + AREA_ATOL).all()), float((area - ref).abs().max())
    again = torch.empty_like(area)
    nat.mask_stats(masks, oh, ow, again, None)
    assert torch.equal(again, area)  # deterministic across calls, bit for bit
    if n > 2:
        assert torch.equal(area[0], area[1])  # equal masks, equal areas


def torch_scored(masks, score, oh, ow, kept_only):
    v = torch_resized(masks, oh, ow)
    n = masks.shape[0]
    scored = torch.cat([torch.full((1, oh, ow), 0.1, device='cuda'), v * score[:, None, None]])
    hard = scored.argmax(0)
    own = torch.cat([torch.zeros((1, oh, ow), device='cuda'), v]).gather(0, hard[None])[0]
    keep = (hard > 0) & (own >= 0.5)
    won = torch.bincount(hard.flatten(), minlength=n + 1)
    kept = torch.bincount(hard[keep], minlength=n + 1)
    return (torch.where(keep, hard, 0) if kept_only else hard), won, kept


@pytest.mark.parametrize('n,size', [(0, SIZES[1]), (1, SIZES[1]), (2, SIZES[5]), (33, SIZES[3]), (257, SIZES[4]),
                                    (1500, SIZES[1]), (4500, SIZES[1]), (31, SIZES[2]), (33, SIZES[0])])
@pytest.mark.parametrize('suppress', [True, False])
def test_scored_argmax_matches_torch(nat, n, size, suppress):
    """n = 4500 puts the 2 (n + 1) counters past the shared-memory limit: the global-counter path."""
    (h, w), (oh, ow) = size
    masks = random_masks(n, h, w, seed=7 * n + oh)
    area = torch.empty(n, device='cuda')
    nat.mask_stats(masks, oh, ow, area, None)
    score = area if suppress else area.max() * 2 - area if n else area
    slot = torch.empty((oh, ow), dtype=torch.int32, device='cuda')
    won = torch.empty(n + 1, dtype=torch.int32, device='cuda')
    kept = torch.empty_like(won)
    nat.mask_scored_argmax(masks.view(torch.uint8), oh, ow, score, suppress, slot, won, kept)
    ref_slot, ref_won, ref_kept = torch_scored(masks, score, oh, ow, suppress)
    assert torch.equal(slot.long(), ref_slot)
    assert torch.equal(won.long(), ref_won) and torch.equal(kept.long(), ref_kept)


@pytest.mark.parametrize('n,size', [(0, SIZES[1]), (1, SIZES[1]), (5, SIZES[5]), (20, SIZES[3]), (50, SIZES[4]),
                                    (257, SIZES[6]), (9000, SIZES[1]), (33, SIZES[0]), (31, SIZES[2])])
def test_last_cover_matches_torch(nat, n, size):
    """n = 9000 counters do not fit in shared memory: the global-counter path."""
    (h, w), (oh, ow) = size
    masks = random_masks(n, h, w, seed=11 * n + ow)
    order = torch.randperm(n, generator=torch.Generator().manual_seed(n)).to(torch.int32).cuda()
    slot = torch.empty((oh, ow), dtype=torch.int32, device='cuda')
    covered = torch.empty(n, dtype=torch.int32, device='cuda')
    nat.mask_last_cover(masks, oh, ow, order, slot, covered)
    on = torch_resized(masks, oh, ow) > 0.5
    ref = torch.zeros((oh, ow), dtype=torch.long, device='cuda')
    for k in order.tolist():
        ref[on[k]] = k + 1
    assert torch.equal(slot.long(), ref)
    assert torch.equal(covered.long(), on.flatten(1).sum(1))


@pytest.fixture(scope='module')
def golden(golden_dir):
    meta = json.load(open(os.path.join(golden_dir, 'detector_masks.json')))
    return meta, dict(np.load(os.path.join(golden_dir, 'detector_masks.npz')))


def test_auto_segment_matches_reference(nat, sc, golden):
    from deva.ext.automatic_sam import auto_segment
    meta, arrays = golden
    for case, rec in zip(sc.AUTO_CASES, meta['auto']):
        name, (h, w), min_side, suppress, thr, fwd, spec = case
        masks = sc.build_masks(spec, h, w, rec['seed'])
        sam = sc.FakeAutoSam(masks, sc.iou_preds(len(masks), rec['seed']), 'cuda')
        fm = sc.forward_mask(fwd, h, w)
        out, segs = auto_segment(sc.auto_config(thr), sam, sc.image(h, w), None if fm is None else fm.cuda(), min_side,
                                 suppress)
        assert out.dtype == torch.int64 and out.is_cuda, name
        np.testing.assert_array_equal(out.cpu().numpy(), arrays[f'auto_{name}'], err_msg=name)
        assert sc.segments_json(segs) == rec['segments'], name
        assert len(sam.calls) == len(rec['calls']), name
        for got, want in zip(sam.calls, rec['calls']):  # generate(image, positive points, None): points from torch
            assert got[:3] == want[:3], name
            assert len(got[3]) == len(want[3]), name
            for a, b in zip(got[3], want[3]):
                assert (a is None and b is None) or np.allclose(a, b, rtol=0, atol=1e-6), name


def test_segment_with_text_matches_reference(nat, sc, golden):
    from deva.ext.grounding_dino import segment_with_text
    meta, arrays = golden
    for case, rec in zip(sc.TEXT_CASES, meta['text']):
        name, (h, w), min_side, nms, boxes = case
        gd, sam = sc.FakeGroundingDino(boxes, 'cuda'), sc.FakeSamPredictor()
        out, segs = segment_with_text(sc.text_config(nms), gd, sam, sc.image(h, w), ['a', 'b'], min_side)
        assert out.dtype == torch.int64 and out.is_cuda, name
        np.testing.assert_array_equal(out.cpu().numpy(), arrays[f'text_{name}'], err_msg=name)
        assert sc.segments_json(segs) == rec['segments'], name
        assert json.loads(json.dumps(gd.calls + sam.calls)) == rec['calls'], name


def _syncs(fn):
    """-> where each host synchronisation of fn() came from, (file, line)."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode('default')
    return [(os.path.basename(w.filename), w.lineno) for w in caught
            if 'called a synchronizing CUDA operation' in str(w.message)]  # not the mode's one-time prototype notice


def test_each_call_synchronises_once(nat, sc):
    from deva.ext.automatic_sam import auto_segment
    from deva.ext.grounding_dino import segment_with_text
    h, w = 1080, 1920
    masks = sc.build_masks([('rand', 32)], h, w, 3)
    img = sc.image(h, w)
    for suppress in (True, False):
        sam = sc.FakeAutoSam(masks, sc.iou_preds(32, 3), 'cuda')
        auto_segment(sc.auto_config(0.8), sam, img, None, 480, suppress)  # warm-up
        syncs = _syncs(lambda: auto_segment(sc.auto_config(0.8), sam, img, None, 480, suppress))
        assert len(syncs) == 1, syncs
    boxes = sc.TEXT_CASES[-1][4]
    segment_with_text(sc.text_config(0.8), sc.FakeGroundingDino(boxes, 'cuda'), sc.FakeSamPredictor(), img, ['a'], 480)
    syncs = _syncs(lambda: segment_with_text(sc.text_config(0.8), sc.FakeGroundingDino(boxes, 'cuda'),
                                             sc.FakeSamPredictor(), img, ['a'], 480))
    assert len(syncs) == 1, syncs
