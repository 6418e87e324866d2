"""The device mask generator's CPU side: oracle/sam_masks.py against the reference generator's fixture
(tests/golden/sam_masks.{json,npz}, minted by make_sam_masks_golden.py), the stand-in segment_anything against the real
package where it is installed, and deva.ext.sam_masks importing without segment_anything or CUDA."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
sys.path.insert(0, GOLDEN)

import sam_masks_scenario as sc  # noqa: E402
from make_sam_masks_golden import digest  # noqa: E402
from oracle import sam_masks, sam_stub  # noqa: E402

META = json.load(open(os.path.join(GOLDEN, 'sam_masks.json')))
ARRAYS = np.load(os.path.join(GOLDEN, 'sam_masks.npz'))


def test_fixture_covers_every_case():
    assert set(META) == set(sc.CASES)
    assert any(m.get('error') for m in META.values())  # the empty positive set
    assert any(m.get('masks', [0, [1]])[1][0] == 0 for m in META.values() if 'masks' in m)  # a frame with no masks
    assert {m['boxes'][0] for m in META.values() if 'boxes' in m} == {'int64', 'float32'}
    assert any(np.isnan(ARRAYS[f'{c}/stability_bits'].view(np.float32)).any() for c in META if 'masks' in META[c])


@pytest.mark.parametrize('case', sorted(sc.CASES))
def test_oracle_matches_reference_fixture(case):
    mk, gk, img, pos, neg = sc.arguments(case)
    want = META[case]
    if 'error' in want:
        with pytest.raises(ValueError):
            sam_masks.generate(sam_stub.FakeSam(**mk), img, **gk, positive_points=pos, negative_points=neg)
        return
    out = sam_masks.generate(sam_stub.FakeSam(**mk), img, **gk, positive_points=pos, negative_points=neg)
    for k in ('masks', 'iou_preds', 'points', 'stability_score', 'boxes'):
        assert [str(out[k].dtype).replace('torch.', ''), list(out[k].shape)] == want[k], k
    np.testing.assert_array_equal(out['iou_preds'].numpy(), ARRAYS[f'{case}/iou_preds'])
    np.testing.assert_array_equal(out['points'].numpy(), ARRAYS[f'{case}/points'])
    np.testing.assert_array_equal(out['stability_score'].view(torch.int32).numpy(), ARRAYS[f'{case}/stability_bits'])
    np.testing.assert_array_equal(out['boxes'].numpy(), ARRAYS[f'{case}/boxes'])
    np.testing.assert_array_equal(out['masks'].flatten(1).sum(1).numpy(), ARRAYS[f'{case}/areas'])
    assert digest(out['masks']) == want['mask_sha256']


def test_fake_model_straddles_the_thresholds():
    """Predicted IoUs straddle 0.88 and tie; stability scores straddle 0.95."""
    mk, gk, img, _, _ = sc.arguments('grid16_thresholds')
    out = sam_masks.generate(sam_stub.FakeSam(**mk), img, **gk)
    iou, stab = out['iou_preds'], out['stability_score']
    assert (iou < 0.88).any() and (iou > 0.88).any() and len(set(iou.tolist())) < iou.numel()
    assert (stab < 0.95).any() and (stab >= 0.95).any()


def test_module_imports_without_segment_anything_or_cuda():
    code = ('import sys, torch\n'
            'import deva.ext.sam_masks, deva.ext.automatic_sam\n'
            'assert not any(m.startswith("segment_anything") for m in sys.modules)\n'
            'assert not torch.cuda.is_initialized()\n')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, 'tracking-anything-with-deva_b200'), ROOT]))
    subprocess.run([sys.executable, '-c', code], check=True, env=env)


def test_switch_rejects_unknown_generator():
    sys.path.insert(0, os.path.join(ROOT, 'tracking-anything-with-deva_b200'))
    from deva.ext.automatic_sam import get_sam_model
    with pytest.raises(ValueError):
        get_sam_model({'sam_variant': 'original'}, 'cpu', mask_generator='cpu')


def test_device_generator_rejects_frames_the_counters_cannot_hold():
    sys.path.insert(0, os.path.join(ROOT, 'tracking-anything-with-deva_b200'))
    saved = sam_stub.install()
    try:
        from deva.ext.sam_masks import DeviceMaskGenerator, point_grid
        gen = DeviceMaskGenerator(sam_stub.FakeSam(), 4, 4, 0.88)
        with pytest.raises(ValueError):
            gen.generate(np.zeros((2, 32768, 3), dtype=np.uint8))
        with pytest.raises(ValueError):
            gen.generate(np.zeros((8, 8, 3), dtype=np.uint8), np.zeros((0, 2), dtype=np.float32))
        np.testing.assert_array_equal(point_grid(7), sam_stub.build_point_grid(7))
    finally:
        sam_stub.uninstall(saved)


def test_stub_matches_segment_anything():
    """The restated helpers against the real package, where it is installed."""
    pytest.importorskip('segment_anything')
    from segment_anything.utils import amg
    from segment_anything.utils.transforms import ResizeLongestSide
    g = torch.Generator().manual_seed(0)
    masks = torch.randn(5, 37, 53, generator=g) * 3
    masks[1] = -5
    for off in (1.0, 0.5):
        torch.testing.assert_close(sam_stub.calculate_stability_score(masks, 0.0, off),
                                   amg.calculate_stability_score(masks, 0.0, off), equal_nan=True, rtol=0, atol=0)
    assert torch.equal(sam_stub.batched_mask_to_box(masks > 0), amg.batched_mask_to_box(masks > 0))
    assert np.array_equal(sam_stub.build_point_grid(9), amg.build_point_grid(9))
    assert sam_stub.generate_crop_boxes((480, 640), 0, 512 / 1500) == amg.generate_crop_boxes((480, 640), 0, 512 / 1500)
    pts = np.random.default_rng(0).uniform(0, 500, (7, 3, 2))
    assert np.array_equal(sam_stub.ResizeLongestSide(1024).apply_coords(pts, (333, 517)),
                          ResizeLongestSide(1024).apply_coords(pts, (333, 517)))
    from segment_anything.modeling import Sam
    low = torch.randn(2, 3, 256, 256, generator=g)
    fake = sam_stub.FakeSam()
    assert torch.equal(fake.postprocess_masks(low, (664, 1024), (333, 517)),
                       Sam.postprocess_masks(fake, low, (664, 1024), (333, 517)))
