"""Resized frame / mask ingest (frame_io.frame_from_rgb8(size=...), mask_from_index8) on the device, against torch on the
CPU, PIL's nearest maps and fixtures recorded from the unmodified reference by
tests/golden/make_ingest_golden.py."""
import io
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _torch_cpu(frame_u8, oh, ow, antialias, flip):
    """The reference's CPU arithmetic: ToTensor (x / 255) and Normalize, then F.interpolate, then the driver's flip."""
    from deva.inference.frame_io import IMAGENET_MEAN, IMAGENET_STD
    x = frame_u8.permute(2, 0, 1).float().div(255)
    x = (x - torch.tensor(IMAGENET_MEAN).view(3, 1, 1)) / torch.tensor(IMAGENET_STD).view(3, 1, 1)
    if (oh, ow) != tuple(x.shape[1:]):
        x = F.interpolate(x[None], (oh, ow), mode='bilinear', align_corners=False, antialias=antialias)[0]
    return torch.flip(x, dims=[-1]) if flip else x


@pytest.mark.parametrize('h,w,size', [(1080, 1920, 480), (2160, 3840, 480), (720, 1280, 480), (480, 854, 240),
                                      (480, 854, 720), (97, 131, 60), (131, 97, 301)])
@pytest.mark.parametrize('resize', ['reader', 'demo'])
@pytest.mark.parametrize('flip', [False, True])
def test_resized_ingest_matches_torch_cpu(h, w, size, resize, flip):
    from deva.inference.frame_io import demo_size, frame_from_rgb8, reader_size
    g = torch.Generator().manual_seed(h * 7 + w)
    frame = torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8)
    out = frame_from_rgb8(frame.pin_memory(), size=size, resize=resize, flip=flip)
    oh, ow = (reader_size if resize == 'reader' else demo_size)(h, w, size)
    ref = _torch_cpu(frame, oh, ow, resize == 'reader', flip)
    assert out.shape == ref.shape
    err = float((out.cpu() - ref).abs().max())
    exact = float((out.cpu() == ref).float().mean())
    print(f'{h}x{w} -> {oh}x{ow} {resize} flip={flip}: max |device - torch CPU| = {err:.2e}, bit-exact fraction {exact:.4f}')
    assert err <= TOL


def test_same_size_is_todays_ingest_bit_for_bit():
    from deva.inference.frame_io import frame_from_rgb8
    g = torch.Generator().manual_seed(3)
    frame = torch.randint(0, 256, (480, 854, 3), generator=g, dtype=torch.uint8).pin_memory()
    plain = frame_from_rgb8(frame)
    for resize in ('reader', 'demo'):
        assert torch.equal(frame_from_rgb8(frame, size=480, resize=resize), plain)
        assert torch.equal(frame_from_rgb8(frame, size=480, resize=resize, flip=True), torch.flip(plain, dims=[-1]))
    assert torch.equal(frame_from_rgb8(frame, flip=True), torch.flip(plain, dims=[-1]))


def test_vipseg_frame_matches_reference_readers(golden_dir):
    from PIL import Image
    from deva.inference.frame_io import frame_from_rgb8
    g = np.load(os.path.join(golden_dir, 'ingest_vipseg.npz'))
    decoded = np.array(Image.open(io.BytesIO(g['jpeg'].tobytes())).convert('RGB'))  # the reader's decode
    assert np.array_equal(decoded[::16, ::16], g['decoded_lattice']), 'PIL decodes the JPEG differently here'
    frame = torch.from_numpy(decoded).pin_memory()
    for resize in ('reader', 'demo'):
        out = frame_from_rgb8(frame, size=480, resize=resize).cpu()
        assert tuple(out.shape) == tuple(g[f'{resize}_shape'])
        err = float((out[:, ::8, ::8] - torch.from_numpy(g[f'{resize}_lattice'])).abs().max())
        print(f'vipseg 1280x720 -> {tuple(out.shape[1:])} {resize}: max |device - reference| = {err:.2e}')
        assert err <= TOL


def test_mask_ingest_matches_reference_reader(golden_dir):
    from deva.inference.frame_io import mask_from_index8
    c1 = np.load(os.path.join(golden_dir, 'config1_vos.npz'))
    ref = torch.from_numpy(np.load(os.path.join(golden_dir, 'ingest_vos240.npz'))['mask0'].astype(np.int64))
    mask = torch.from_numpy(c1['mask0'])
    out = mask_from_index8(mask, 240)
    assert out.dtype == torch.long and torch.equal(out.cpu(), ref)
    assert torch.equal(mask_from_index8(mask, 240, flip=True).cpu(), torch.flip(ref, dims=[-1]))
    assert torch.equal(mask_from_index8(mask).cpu(), mask.long())


@pytest.mark.parametrize('h,w,size', [(480, 854, 720), (97, 131, 60), (131, 97, 301), (1080, 1920, 480), (3, 5, 11)])
@pytest.mark.parametrize('flip', [False, True])
def test_mask_ingest_is_the_pinned_gather(h, w, size, flip):
    from deva.inference.frame_io import mask_from_index8, pil_nearest_map, reader_size
    g = torch.Generator().manual_seed(h + w)
    mask = torch.randint(0, 256, (h, w), generator=g, dtype=torch.uint8)
    oh, ow = reader_size(h, w, size)
    ref = mask.long()[torch.from_numpy(pil_nearest_map(h, oh)).long()][:, torch.from_numpy(pil_nearest_map(w, ow)).long()]
    if flip:
        ref = torch.flip(ref, dims=[-1])
    assert torch.equal(mask_from_index8(mask.cuda(), size, flip=flip).cpu(), ref)


@pytest.mark.parametrize('flip', [False, True])
def test_size_240_session_matches_reference(golden_dir, synthetic_sd, flip):
    """example/vos/bmx-trees at --size 240 driven like evaluation/eval_vos.py:133-198: uint8 frame -> resized ingest
    (+ flip) -> step -> prob_to_ids(resize back to 480x854, flip back), with the contract and structure of
    test_config1_gpu.py."""
    from deva.inference.frame_io import frame_from_rgb8, mask_from_index8, prob_to_ids
    from deva.inference.inference_core import DEVAInferenceCore
    from deva.model.network import DEVA
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    tol = 1e-3
    c1 = np.load(os.path.join(golden_dir, 'config1_vos.npz'))
    g = np.load(os.path.join(golden_dir, 'ingest_vos240.npz'))
    meta = json.load(open(os.path.join(golden_dir, 'ingest_vos240.json')))
    tag = 'flip' if flip else 'noflip'
    lattice = meta['lattice']
    cfg = meta['runs'][tag]
    net = DEVA(cfg).cuda().eval()
    net.load_weights({k: v.cuda() for k, v in synthetic_sd.items()})
    np.random.seed(42)
    core = DEVAInferenceCore(net, cfg)
    frames = torch.from_numpy(c1['frames_u8'])
    T, (H, W) = frames.shape[0], frames.shape[1:3]
    worst, over = 0.0, 0.0
    for t in range(T):
        img = frame_from_rgb8(frames[t].pin_memory(), size=meta['size'], flip=flip)
        if t == 0:
            assert tuple(img.shape) == tuple(g['image0_shape'])
            unflipped = torch.flip(img, dims=[-1]) if flip else img  # the reader's output comes before the driver's flip
            assert float((unflipped.cpu()[:, ::lattice, ::lattice] - torch.from_numpy(g['image0_lattice'])).abs().max()) <= TOL
            mask = mask_from_index8(torch.from_numpy(c1['mask0']), meta['size'], flip=flip)
            p = core.step(img, mask, meta['labels'])
        else:
            p = core.step(img, end=(t == T - 1))
        assert tuple(p.shape) == (len(meta['labels']) + 1, 240, 427)
        ids = prob_to_ids(p.float(), core.object_manager, size=(H, W), flip=flip, dtype=torch.uint8).cpu()
        ref_ids = torch.from_numpy(g[f'{tag}_ids_{t}'])
        assert set(ids.unique().tolist()) <= {0, *meta['labels']}
        confident = torch.from_numpy(np.unpackbits(g[f'{tag}_confident_{t}'])[:H * W].reshape(H, W).astype(bool))
        assert bool((ids[confident] == ref_ids[confident]).all()), t
        lat = torch.from_numpy(g[f'{tag}_prob_lattice_{t}'])
        got = p.float().cpu()[:, ::lattice, ::lattice]
        d = (got - lat).abs()
        worst = max(worst, float(d.max()))
        over = max(over, float((d > tol).float().mean()))
        top2 = torch.topk(lat, 2, dim=0)[0]
        decided = (top2[0] - top2[1]) > 2 * max(tol, float(d.max()))
        assert bool((got.argmax(0)[decided] == lat.argmax(0)[decided]).all()), t
        assert float(decided.float().mean()) > 0.5 or t > 0
    print(f'[size 240, {tag}] example/vos clip: max |prob - reference| on the lattice = {worst:.3e}, fraction of lattice '
          f'points over {tol:g}: {over:.2e}')
    assert over <= 5e-4, (over, worst)
    assert worst < 3e-3, worst
