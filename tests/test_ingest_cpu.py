"""Host side of the resized frame / mask ingest (deva/inference/frame_io.py): output-size rules, PIL's nearest index maps
and the resampling weight tables, against torchvision, PIL and torch on the CPU."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image
from torchvision import transforms

from deva.inference import frame_io as fio

SHAPES = [(480, 854), (720, 1280), (1080, 1920), (2160, 3840), (854, 480), (480, 480), (97, 131), (131, 97), (360, 641),
          (1001, 999)]
SIZES = [240, 480, 720, 97]


@pytest.mark.parametrize('h,w', SHAPES)
def test_reader_size_is_torchvision_resize(h, w):
    for size in SIZES:
        out_w, out_h = transforms.Resize(size, interpolation=transforms.InterpolationMode.NEAREST)(Image.new('L', (w, h))).size
        assert fio.reader_size(h, w, size) == (out_h, out_w), (h, w, size)


@pytest.mark.parametrize('h,w', SHAPES)
def test_demo_size_is_demo_utils_expression(h, w):
    for size in SIZES:
        scale = size / min(h, w)  # deva/inference/demo_utils.py:15-16
        assert fio.demo_size(h, w, size) == (int(h * scale), int(w * scale))


def test_demo_size_non_integer_scale():
    assert fio.demo_size(720, 1280, 480) == (480, 853)
    assert fio.reader_size(720, 1280, 480) == (480, 853)


@pytest.mark.parametrize('h,w', SHAPES)
def test_nearest_maps_are_pil(h, w):
    """Resizing an index ramp with PIL's NEAREST reveals the source index of every output row and column."""
    ramp_x = Image.fromarray(np.arange(w, dtype=np.int32)[None], mode='I')
    ramp_y = Image.fromarray(np.arange(h, dtype=np.int32)[:, None], mode='I')
    for size in SIZES:
        oh, ow = fio.reader_size(h, w, size)
        assert np.array_equal(np.array(ramp_x.resize((ow, 1), Image.NEAREST))[0], fio.pil_nearest_map(w, ow)), (w, ow)
        assert np.array_equal(np.array(ramp_y.resize((1, oh), Image.NEAREST))[:, 0], fio.pil_nearest_map(h, oh)), (h, oh)


def test_nearest_maps_resize_a_mask_like_pil():
    g = np.random.default_rng(0)
    for h, w, oh, ow in [(480, 854, 720, 1281), (97, 131, 60, 81), (97, 131, 301, 407)]:
        mask = g.integers(0, 7, (h, w), dtype=np.uint8)
        ref = np.array(Image.fromarray(mask).convert('P').resize((ow, oh), Image.NEAREST))
        got = mask[fio.pil_nearest_map(h, oh)][:, fio.pil_nearest_map(w, ow)]
        assert np.array_equal(got, ref)


def _normalised(frame_u8):
    x = torch.from_numpy(frame_u8).permute(2, 0, 1).float().div(255)
    return (x - torch.tensor(fio.IMAGENET_MEAN).view(3, 1, 1)) / torch.tensor(fio.IMAGENET_STD).view(3, 1, 1)


def _emulate_kernel(x, taps_fn, oh, ow):
    """numpy model of the two passes of deva_b200_ingest_rgb8_resize: horizontal, then vertical, each a chain of fp32
    fused multiply-adds in tap order (an fp64 product plus fp64 add rounded to fp32 stands for the fused operation)."""
    def one_axis(v, idx, wt):
        acc = np.zeros(v.shape[:-1] + (idx.shape[0],), np.float32)
        for j in range(idx.shape[1]):
            acc = (v[..., idx[:, j]].astype(np.float64) * wt[:, j] + acc).astype(np.float32)
        return acc
    c, h, w = x.shape
    rows = one_axis(x, *taps_fn(w, ow))
    return np.swapaxes(one_axis(np.swapaxes(rows, 1, 2), *taps_fn(h, oh)), 1, 2)


@pytest.mark.parametrize('h,w,oh,ow', [(1080, 1920, 480, 853), (720, 1280, 480, 853), (480, 854, 240, 427),
                                       (480, 854, 720, 1281), (97, 131, 60, 81), (131, 97, 301, 200), (480, 854, 480, 300)])
@pytest.mark.parametrize('antialias', [True, False])
def test_weight_tables_match_torch_cpu(h, w, oh, ow, antialias):
    frame = np.random.default_rng(h * w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    x = _normalised(frame)
    ref = F.interpolate(x[None], (oh, ow), mode='bilinear', align_corners=False, antialias=antialias)[0].numpy()
    got = _emulate_kernel(x.numpy(), fio.antialias_taps if antialias else fio.bilinear_taps, oh, ow)
    err = float(np.abs(got - ref).max())
    print(f'{h}x{w} -> {oh}x{ow} antialias={antialias}: max |emulated kernel - torch CPU| = {err:.2e}')
    assert err <= 1e-5


def test_weight_tables_shape_and_normalisation():
    idx, wt = fio.antialias_taps(3840, 853)
    assert idx.dtype == np.int32 and wt.dtype == np.float32 and idx.shape == wt.shape == (853, 11)
    assert idx.min() >= 0 and idx.max() < 3840
    assert np.allclose(wt.sum(1), 1, atol=1e-6)
    idx, wt = fio.bilinear_taps(480, 480)  # same size: the identity
    assert np.array_equal(idx[:, 0], np.arange(480)) and np.array_equal(wt, np.stack([np.ones(480), np.zeros(480)], 1))
