"""GPU: the SAM mask kernels (csrc/sam_masks.cu) against torch's two-stage F.interpolate and torchvision's batched_nms
on CUDA, and DeviceMaskGenerator / auto_segment against the unmodified reference generator (staged under
oracle/_ref by oracle/build_ref_sam.py), run live on the same GPU over oracle/sam_stub.py's stand-in segment_anything
and FakeSam."""
import importlib.util
import os
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def nat():
    from deva import _native
    _native.require_device()
    return _native


@pytest.fixture(scope='module')
def sc(golden_dir):
    spec = importlib.util.spec_from_file_location('sam_masks_scenario', os.path.join(golden_dir, 'sam_masks_scenario.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module')
def stub():
    from oracle import sam_masks, sam_stub
    if not sam_masks.reference_available():
        pytest.fail('oracle/_ref/deva/ext/SAM is not staged (oracle/build_ref_sam.py)')
    saved = sam_stub.install()
    yield sam_stub, sam_masks.reference_generator()
    sam_stub.uninstall(saved)


def input_size(h, w):
    s = 1024 / max(h, w)
    return int(h * s + 0.5), int(w * s + 0.5)


def smooth_logits(n, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 1, 16, 16, generator=g) * 6
    x = F.interpolate(x, (256, 256), mode='bicubic', align_corners=False)[:, 0]
    x[0] = -3  # entirely below -1
    return x.contiguous().cuda()


def torch_stats(v, thr=0.0, off=1.0):
    m = v > thr
    st = torch.zeros(v.shape[0], 7, dtype=torch.int64)
    st[:, 0] = (v > thr + off).flatten(1).sum(1).cpu()
    st[:, 1] = (v > thr - off).flatten(1).sum(1).cpu()
    st[:, 2] = m.flatten(1).sum(1).cpu()
    for j in range(v.shape[0]):
        ys, xs = torch.nonzero(m[j].any(1)), torch.nonzero(m[j].any(0))
        st[j, 3:] = torch.tensor([xs.min(), ys.min(), xs.max(), ys.max()]) if len(ys) else torch.tensor([2**31 - 1] * 2 + [-1] * 2)
    return st


SHAPES = [(1, 1), (1, 7), (5, 1), (480, 640), (300, 200), (333, 517), (720, 1280), (1080, 1920), (17, 1000),
          (1000, 3), (1024, 1024), (2048, 1536), (2160, 3840)]


@pytest.mark.parametrize('h,w', SHAPES)
def test_stats_and_masks_match_torch(nat, h, w):
    from oracle.sam_masks import upsample
    n = 6 if h * w < 4e6 else 2
    logits = smooth_logits(n, h * 7 + w)
    ih, iw = input_size(h, w)
    v = upsample(logits, 1024, (ih, iw), (h, w))  # torch's CUDA F.interpolate, as Sam.postprocess_masks calls it
    stats = torch.empty(n, 7, dtype=torch.int32, device='cuda')
    nat.sam_mask_stats(logits, 1024, ih, iw, h, w, None, 0.0, 1.0, -1.0, 0.0, stats)
    masks = torch.empty(n, h, w, dtype=torch.bool, device='cuda')
    nat.sam_mask_write(logits, torch.arange(n, device='cuda'), 1024, ih, iw, h, w, 0.0, masks)
    want = torch_stats(v)
    got = stats.cpu().long()
    if not torch.equal(got, want) or not torch.equal(masks, v > 0):
        diff = (masks != (v > 0))
        near = min(float(v[diff].abs().min()) if diff.any() else 1.0, 1.0)
        pytest.fail(f'{h}x{w}: stats differ in {(got != want).sum().item()} fields, masks in {diff.sum().item()} '
                    f'pixels (closest to the threshold: {near:.3e})\n{got}\n{want}')


def test_stats_skip_masks_below_the_iou_threshold(nat):
    logits = smooth_logits(4, 1)
    iou = torch.tensor([0.9, 0.88, 0.5, 0.95], device='cuda')
    stats = torch.empty(4, 7, dtype=torch.int32, device='cuda')
    nat.sam_mask_stats(logits, 1024, 768, 1024, 480, 640, iou, 0.88, 1.0, -1.0, 0.0, stats)
    st = stats.cpu()
    assert st[1, :3].tolist() == [0, 0, 0] and st[2, :3].tolist() == [0, 0, 0] and st[3, 1] > 0
    stab = torch.empty(4, device='cuda')
    boxes = torch.empty(4, 4, dtype=torch.int64, device='cuda')
    kept = torch.empty(5, dtype=torch.int32, device='cuda')
    nat.sam_mask_compact(stats, iou, 0.88, 0.0, stab, boxes, kept)
    assert kept.cpu().tolist()[:3] == [2, 0, 3]
    assert torch.isnan(stab[0]) and boxes[0].tolist() == [0, 0, 0, 0]  # the mask entirely below -1


def nms_cases():
    g = torch.Generator().manual_seed(0)
    for n in (0, 1, 2, 300, 3000):
        xy = torch.randint(0, 200, (n, 2), generator=g)
        wh = torch.randint(0, 60, (n, 2), generator=g)
        boxes = torch.cat([xy, xy + wh], 1).float()
        scores = torch.randint(0, 8, (n,), generator=g).float() / 8  # many ties
        yield boxes, scores, 0.7
    # IoU exactly at the threshold: 50 / 100 is not suppressed at 0.5, and is at 0.49
    boxes = torch.tensor([[0, 0, 10, 10], [0, 0, 10, 5], [0, 5, 10, 10], [0, 0, 10, 10]], dtype=torch.float32)
    scores = torch.tensor([0.9, 0.9, 0.9, 0.9])
    yield boxes, scores, 0.5
    yield boxes, scores, 0.49


def test_nms_matches_torchvision(nat):
    from torchvision.ops import batched_nms
    for boxes, scores, thr in nms_cases():
        boxes, scores = boxes.cuda(), scores.cuda()
        want = batched_nms(boxes, scores, torch.zeros(len(scores), dtype=torch.int64, device='cuda'), thr)
        keep = torch.empty(max(len(scores), 1), dtype=torch.int64, device='cuda')
        n_keep = torch.empty(1, dtype=torch.int32, device='cuda')
        nat.sam_nms(boxes, scores, thr, keep, n_keep)
        assert torch.equal(keep[:int(n_keep.item())], want), (len(scores), thr)


def same(a, b):
    if a.dtype != b.dtype or a.shape != b.shape or a.device != b.device:
        return False
    if a.is_floating_point():
        return torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a[~torch.isnan(a)], b[~torch.isnan(b)])
    return torch.equal(a, b)


def test_generate_matches_reference_live(nat, sc, stub):
    from deva.ext.sam_masks import DeviceMaskGenerator
    sam_stub, RefGen = stub
    for case in sc.CASES:
        mk, gk, img, pos, neg = sc.arguments(case)
        model = sam_stub.FakeSam(**mk).cuda()
        dev = DeviceMaskGenerator(model, **gk)
        if pos is not None and len(pos) == 0:
            with pytest.raises(ValueError):
                dev.generate(img, pos, neg)
            continue
        ref = RefGen(model, **gk).generate(img, pos, neg)
        out = dev.generate(img, pos, neg)
        for k in ('masks', 'iou_preds', 'points', 'stability_score', 'boxes'):
            assert same(out[k], ref[k]), (case, k, out[k].dtype, ref[k].dtype, out[k].shape, ref[k].shape)


def _syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode('default')
    return [(os.path.basename(w.filename), w.lineno) for w in caught
            if 'called a synchronizing CUDA operation' in str(w.message)]


def test_generate_synchronises_once_per_batch_and_allocates_no_float_frame(nat, sc, stub):
    from deva.ext.sam_masks import DeviceMaskGenerator
    sam_stub, _ = stub
    h, w = 1080, 1920
    img = sc.image(h, w, 0)
    model = sam_stub.FakeSam(seed=3).cuda()
    gen = DeviceMaskGenerator(model, 32, 64, 0.88)
    out = gen.generate(img)  # warm-up
    batches = (32 * 32 + 63) // 64
    syncs = [s for s in _syncs(lambda: gen.generate(img)) if s[0] == 'sam_masks.py']
    assert len(syncs) <= batches + 1, syncs
    del out
    base = {}
    set_image = gen.predictor.set_image

    def set_image_then_reset_peak(image):  # the image encoder's input is not the generator's to account for
        set_image(image)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base['bytes'] = torch.cuda.memory_allocated()

    gen.predictor.set_image = set_image_then_reset_peak
    # the fake decoder's own float64 temporaries for one batch are the model's, not the generator's
    gen.predictor.set_image(img)
    gen._decode(gen.point_grid[:64] * np.array([[w, h]]), None, (h, w))
    torch.cuda.synchronize()
    decoder_peak = torch.cuda.max_memory_allocated() - base['bytes']
    out = gen.generate(img)
    peak = torch.cuda.max_memory_allocated() - base['bytes']
    gen.predictor.set_image = set_image
    # live at once: the returned masks, the logits kept before NMS (twice while they are concatenated), one batch's
    # decoder output and its float copy, and small per-mask tensors.  A full-resolution
    # float mask (h * w * 4 bytes) on top of that would exceed the slack.
    logit_bytes = 256 * 256 * 4
    bound = (out['masks'].numel() + 2 * gen.candidates * logit_bytes + 2 * 3 * 64 * logit_bytes + decoder_peak
             + (1 << 21))
    print(f'peak extra {peak / 2**20:.1f} MiB (bound {bound / 2**20:.1f} MiB) for {gen.candidates} candidates; '
          f'one float frame is {h * w * 4 / 2**20:.1f} MiB')
    assert gen.candidates > 0 and peak <= bound
    assert (1 << 21) < h * w * 4


def test_auto_segment_through_get_sam_model(nat, sc, stub):
    import deva.ext
    from deva.ext.automatic_sam import auto_segment, get_sam_model
    ref_ext = os.path.join(ROOT, 'oracle', '_ref', 'deva', 'ext')
    if ref_ext not in deva.ext.__path__:
        deva.ext.__path__.append(ref_ext)  # deva.ext.SAM resolves to the staged reference, as to a reference checkout
    config = {'sam_variant': 'original', 'SAM_ENCODER_VERSION': 'fake', 'SAM_CHECKPOINT_PATH': None,
              'SAM_NUM_POINTS_PER_SIDE': 32, 'SAM_NUM_POINTS_PER_BATCH': 64, 'SAM_PRED_IOU_THRESHOLD': 0.88,
              'SAM_OVERLAP_THRESHOLD': 0.5}
    ref = get_sam_model(config, 'cuda', mask_generator='reference')
    dev = get_sam_model(config, 'cuda', mask_generator='device')
    assert type(dev).__name__ == 'DeviceMaskGenerator' and type(ref).__name__ == 'SamAutomaticMaskGenerator'
    img = sc.image(480, 640, 11)
    fm = torch.zeros(480, 640, dtype=torch.int64, device='cuda')
    fm[100:300, 200:500] = 1
    for forward_mask in (None, fm):
        for suppress in (True, False):
            a_map, a_segs = auto_segment(config, ref, img, forward_mask, 480, suppress)
            b_map, b_segs = auto_segment(config, dev, img, forward_mask, 480, suppress)
            assert torch.equal(a_map, b_map)
            assert [(s.id, s.scores) for s in a_segs] == [(s.id, s.scores) for s in b_segs]
            assert len(a_segs) > 0
