"""Multi-scale / flip evaluation on the device (frame_io.prob_to_scores / scores_to_ids, multi_scale.MultiScaleCore)
against torch and numpy restatements of eval_vos.py --save_scores and scripts/merge_multi_scale.py, and against the
fixture minted from the unmodified reference by tests/golden/make_multiscale_golden.py."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _torch_scores(prob, size, flip):
    """eval_vos.py:169-177, :188-189 on the device: resize back, flip back, (prob * 255) truncated to uint8; also
    returns the float product so a test can tell where a last-bit difference of the resized value matters."""
    ref = prob
    if size is not None:
        ref = F.interpolate(ref.unsqueeze(1), size, mode='bilinear', align_corners=False)[:, 0]
    if flip:
        ref = torch.flip(ref, dims=[-1])
    x = ref * 255
    return x.to(torch.uint8), x


def _numpy_merge(members, mapping):
    """scripts/merge_multi_scale.py::process_vid: float32 sum, np.argmax, the remap loop."""
    total = None
    for s in members:
        total = s.astype(np.float32) if total is None else total + s
    result = np.argmax(total, axis=0)
    if mapping is None:
        return result.astype(np.uint8)
    idx = np.zeros_like(result, dtype=np.uint8)
    for l, i in mapping.items():
        idx[result == i] = l
    return idx


def _prob(k1, h, w, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    prob = torch.softmax(4 * torch.randn(k1, max(h // 8, 1), max(w // 8, 1), device='cuda', generator=g), 0)
    return F.interpolate(prob.unsqueeze(0), size=(h, w), mode='bilinear', align_corners=False)[0].contiguous()


@pytest.mark.parametrize('shape,size,flip', [
    ((6, 120, 216), None, False), ((6, 120, 216), None, True), ((6, 120, 216), (270, 480), False),
    ((6, 120, 216), (1080, 1920), True), ((6, 120, 216), (77, 131), False),
    ((6, 480, 854), (1080, 1920), False), ((6, 480, 854), (1080, 1920), True)])
def test_prob_to_scores_matches_torch(shape, size, flip):
    from deva.inference.frame_io import prob_to_scores
    prob = _prob(*shape, seed=sum(shape))
    ref, x = _torch_scores(prob, size, flip)
    out = prob_to_scores(prob, size, flip)
    assert out.dtype == torch.uint8 and out.shape == ref.shape
    diff = (out.int() - ref.int()).abs()
    if size is None:
        assert torch.equal(out, ref)
        frac = 0.0
    else:
        near_int = (x - x.round()).abs() < 1e-4
        assert int(diff.max()) <= 1
        assert not bool((diff > 0)[~near_int].any()), 'a score differs away from an integer boundary'
        frac = float((diff > 0).float().mean())
    print(f'{tuple(shape)} -> {size} flip={flip}: fraction of scores off by 1 from torch {frac:.2e}')
    # the running sum gets exactly the scores, in the same pass, with or without the scores output
    g = torch.Generator(device='cuda').manual_seed(7)
    base = torch.randint(0, 10000, tuple(out.shape), device='cuda', generator=g, dtype=torch.int32)
    into = base.clone()
    again = prob_to_scores(prob, size, flip, into=into)
    assert torch.equal(again, out) and torch.equal(into, base + out.int())
    assert prob_to_scores(prob, size, flip, scores=False, into=into) is None
    assert torch.equal(into, base + 2 * out.int())


@pytest.mark.parametrize('members,c,h,w', [(6, 4, 97, 131), (2, 9, 480, 854), (1, 1, 33, 17), (12, 300, 40, 50)])
def test_scores_to_ids_matches_numpy_merge(members, c, h, w):
    from deva.inference.frame_io import scores_to_ids
    from deva.inference.object_info import ObjectInfo
    from deva.inference.object_manager import ObjectManager
    rng = np.random.default_rng(members * 1000 + c)
    sets = [rng.integers(0, 256, (c, h, w)).astype(np.uint8) for _ in range(members)]
    if c > 1:  # plant exact ties of the top two (and three) channels in every member's scores
        for s in sets:
            s[:, ::3, ::5] = 0
            s[c - 1, ::3, ::5] = 200
            s[c // 2, ::3, ::5] = 200
            s[0, ::6, ::5] = 200
    total = torch.from_numpy(np.stack(sets).sum(0, dtype=np.int32)).cuda()
    om = ObjectManager()
    om.add_new_objects([ObjectInfo(i) for i in (7, 3, 200, 41)][:max(c - 1, 0)])
    mappings = [None, om.get_tmp_to_obj_mapping(), {5: 1, 9: 1, 4: c - 1},  # 9 overwrites 5; other channels unmapped
                {6: 0, 2: c // 2}]  # channel 0 mapped, the rest 0
    for mapping in mappings:
        ref = _numpy_merge(sets, mapping)
        ids = scores_to_ids(total, mapping=mapping).cpu().numpy()
        assert ids.dtype == np.uint8 and np.array_equal(ids, ref), mapping
    assert np.array_equal(scores_to_ids(total, om).cpu().numpy(), _numpy_merge(sets, om.get_tmp_to_obj_mapping()))
    wide = {70000: c - 1, 3: 0}  # an id above 255: only the int64 output holds it
    long_ids = scores_to_ids(total, mapping=wide, dtype=torch.long).cpu().numpy()
    argmax = np.argmax(np.stack(sets).astype(np.float32).sum(0), axis=0)
    last = {i: l for l, i in wide.items()}
    assert np.array_equal(long_ids, np.array([last.get(k, 0) for k in range(c)])[argmax])


def _network(cfg, synthetic_sd):
    from deva.model.network import DEVA
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    net = DEVA(cfg).cuda().eval()
    net.load_weights({k: v.cuda() for k, v in synthetic_sd.items()})
    return net


def _clip(golden_dir):
    c1 = np.load(os.path.join(golden_dir, 'config1_vos.npz'))
    meta = json.load(open(os.path.join(golden_dir, 'multiscale_vos.json')))
    return torch.from_numpy(c1['frames_u8']), torch.from_numpy(c1['mask0']), meta


def _member_scores(net, cfg, frames, mask0, labels, size, flip):
    """eval_vos' loop for one member, by hand: ingest, step, prob_to_scores at the original size."""
    from deva.inference.frame_io import frame_from_rgb8, mask_from_index8, prob_to_scores
    from deva.inference.inference_core import DEVAInferenceCore
    np.random.seed(42)
    core = DEVAInferenceCore(net, dict(cfg))
    T, H, W = frames.shape[:3]
    out = []
    for t in range(T):
        img = frame_from_rgb8(frames[t].pin_memory(), size=size, flip=flip)
        if t == 0:
            p = core.step(img, mask_from_index8(mask0, size, flip=flip), labels)
        else:
            p = core.step(img, end=(t == T - 1))
        out.append(prob_to_scores(p.float(), (H, W), flip))
    return out, core


@pytest.mark.parametrize('member', [(240, True), (None, False)])
def test_one_member_equals_the_eval_vos_loop(golden_dir, synthetic_sd, member):
    from deva.inference.frame_io import scores_to_ids
    from deva.inference.multi_scale import MultiScaleCore
    frames, mask0, meta = _clip(golden_dir)
    net = _network(meta['config'], synthetic_sd)
    ref, core = _member_scores(net, meta['config'], frames, mask0, meta['labels'], *member)
    mapping = core.object_manager.get_tmp_to_obj_mapping()
    np.random.seed(42)
    ms = MultiScaleCore(net, meta['config'], [member])
    T = frames.shape[0]
    for t in range(T):
        if t == 0:
            ids, total = ms.step(frames[t].pin_memory(), mask0, meta['labels'], return_scores=True)
        else:
            ids, total = ms.step(frames[t].pin_memory(), end=(t == T - 1), return_scores=True)
        assert torch.equal(total, ref[t].int()), t
        assert torch.equal(ids, scores_to_ids(ref[t].int(), mapping=mapping)), t
    assert ms.object_manager is ms.cores[0].object_manager
    assert ms.object_manager.get_tmp_to_obj_mapping() == mapping


def test_six_members_match_reference_fixture(golden_dir, synthetic_sd):
    from deva.inference.multi_scale import MultiScaleCore
    frames, mask0, meta = _clip(golden_dir)
    g = np.load(os.path.join(golden_dir, 'multiscale_vos.npz'))
    cfg, labels, step = meta['config'], meta['labels'], meta['lattice']
    members = [(s, bool(f)) for s, f in meta['members']]
    net = _network(cfg, synthetic_sd)
    T, H, W = frames.shape[:3]
    per_member = []
    for m, (size, flip) in enumerate(members):
        scores, _ = _member_scores(net, cfg, frames, mask0, labels, size, flip)
        per_member.append(scores)
        worst, exact = 0, 1.0
        for t in range(T):
            got = scores[t][:, ::step, ::step].int().cpu()
            d = (got - torch.from_numpy(g['scores_lattice'][m, t]).int()).abs()
            worst, exact = max(worst, int(d.max())), min(exact, float((d == 0).float().mean()))
        print(f'member size={size} flip={flip}: max |score - reference| on the lattice = {worst}, '
              f'worst-frame exact fraction {exact:.4f}')
        assert worst <= meta['margin_per_member'], (size, flip)
    np.random.seed(42)
    ms = MultiScaleCore(net, cfg, members)
    decided = torch.from_numpy(np.unpackbits(g['decided'])[:T * H * W].reshape(T, H, W).astype(bool))
    for t in range(T):
        if t == 0:
            ids, total = ms.step(frames[t].pin_memory(), mask0, labels, return_scores=True)
        else:
            ids, total = ms.step(frames[t].pin_memory(), end=(t == T - 1), return_scores=True)
        assert torch.equal(total, sum(s[t].int() for s in per_member)), t
        ids, ref = ids.cpu(), torch.from_numpy(g['ids'][t])
        agree = float((ids == ref).float().mean())
        print(f'frame {t}: decided fraction {float(decided[t].float().mean()):.4f}, merged ids equal the reference on '
              f'{agree:.4f} of all pixels')
        assert bool((ids[decided[t]] == ref[decided[t]]).all()), t
    assert float(decided[0].float().mean()) > 0.5
    assert ms.object_manager.get_tmp_to_obj_mapping() == {int(k): v for k, v in meta['mapping'].items()}


def test_disagreeing_members_and_bad_shapes_raise():
    from deva import _native as nat
    from deva.inference.frame_io import prob_to_scores, scores_to_ids
    from deva.inference.multi_scale import MultiScaleCore
    cfg = dict(key_dim=64, value_dim=512, pix_feat_dim=512, mem_every=5, enable_long_term=True, chunk_size=-1,
               top_k=30, enable_long_term_count_usage=False, max_mid_term_frames=10, min_mid_term_frames=5,
               num_prototypes=128, max_long_term_elements=10000)
    frame = torch.zeros(60, 80, 3, dtype=torch.uint8, device='cuda')

    def fake(channels, order):
        ms = MultiScaleCore(None, cfg, [(None, False), (None, True)])
        for core, c, objs in zip(ms.cores, channels, order):
            core.object_manager.add_new_objects(objs)
            core.step = lambda image, *a, c=c, **k: torch.full((c, *image.shape[1:]), 1.0 / c, device='cuda')
        return ms

    ids = fake((3, 3), ([4, 9], [4, 9])).step(frame)
    assert ids.shape == (60, 80) and bool((ids == 0).all())  # ties: channel 0 (background) wins
    with pytest.raises(RuntimeError, match='channels'):
        fake((3, 4), ([4, 9], [4, 9])).step(frame)
    with pytest.raises(RuntimeError, match='temporary ids'):
        fake((3, 3), ([4, 9], [9, 4])).step(frame)
    with pytest.raises(ValueError):
        fake((3, 3), ([4, 9], [4, 9])).step(frame, torch.zeros(60, 80, dtype=torch.uint8))  # a mask without objects

    prob = _prob(3, 60, 80, seed=1)
    for bad in (torch.zeros(3, 60, 81, dtype=torch.int32, device='cuda'),
                torch.zeros(2, 60, 80, dtype=torch.int32, device='cuda'),
                torch.zeros(3, 60, 80, dtype=torch.int64, device='cuda'),
                torch.zeros(3, 60, 80, dtype=torch.int32)):
        with pytest.raises(RuntimeError):
            prob_to_scores(prob, into=bad)
    with pytest.raises(RuntimeError):
        prob_to_scores(prob, scores=False)
    for bad in (torch.zeros(60, 80, dtype=torch.int32, device='cuda'), torch.zeros(3, 60, 80, device='cuda')):
        with pytest.raises(RuntimeError):
            scores_to_ids(bad)
    with pytest.raises(RuntimeError, match='bad arguments'):  # the library refuses a call with no output
        nat.prob_to_scores(prob, 3, 60, 80, 60, 80, False, None, None)
    with pytest.raises(RuntimeError, match='bad arguments'):
        nat.scores_to_ids(torch.zeros(3, 60, 80, dtype=torch.int32, device='cuda'), 3, 60, 80, None, None, None)
    with pytest.raises(RuntimeError, match='bad arguments'):
        nat.scores_to_ids(torch.zeros(3, 60, 80, dtype=torch.int32, device='cuda'), 0, 60, 80, None, None, None)


def test_export_and_merge_do_not_synchronise():
    from deva.inference.frame_io import prob_to_scores, scores_to_ids
    prob = _prob(6, 480, 854, seed=3)
    total = torch.zeros(6, 1080, 1920, dtype=torch.int32, device='cuda')
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for flip in (False, True):
            prob_to_scores(prob, (1080, 1920), flip, into=total)
        prob_to_scores(prob)
        ids = scores_to_ids(total, mapping={7: 1, 3: 2, 9: 5})
        scores_to_ids(total, dtype=torch.long)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    ref = _numpy_merge([_torch_scores(prob, (1080, 1920), f)[0].cpu().numpy() for f in (False, True)],
                       {7: 1, 3: 2, 9: 5})
    assert float((ids.cpu().numpy() == ref).mean()) > 0.999
