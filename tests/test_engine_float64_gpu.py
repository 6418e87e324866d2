"""The composed native engine (deva/model/native_engine.py) against the oracle network replayed in float64, at the
frame sizes and object counts bench.py times: c2 (480p, 5 objects) and c3 (1080p, 16 objects).

tests/test_stages_gpu.py checks the same stages on a 64 x 80 frame with 2 objects, where every layer is a single edge
tile; here the many-tile schedules, the full-width staged epilogues, the batch-broadcast shared halves across many
objects and the 4x4-pooled head run at the sizes a real video reaches, and the recurrent sensory state is carried over
several decode steps.  Both sides get the same external inputs - frames with real image statistics (the config-1 clip,
upscaled bilinearly for 1080p, ImageNet-normalised and padded to multiples of 16), overlapping soft masks and, as the
memory readout, the oracle's own frame-0 value rounded to fp16 - and each keeps its own features and sensory state.
The oracle (oracle/network.py, pinned to the reference in tests/test_oracle_golden.py) runs one object at a time to
bound its float64 memory: objects never meet before the output tail (quirk Q11).  The bounds are test_stages_gpu.py's;
the one on prob is the engine's contract with the fp32 reference.  Every measured error is printed beside its bound.

Two kinds of row sit beside the bounds:
* regression ceilings (CEILINGS): the measured error plus about 10 %, on the object logits and prob.  They are not
  accuracy contracts; they catch a precision regression of one layer (up_8_4.out_conv in single fp16 moves c3's logits
  from 2.75e-3 to 3.36e-3 and prob from 1.17e-4 to 1.41e-4) long before it reaches a bound.
* a known miss (KNOWN_MISSES): at c3 the background channel of the aggregated logits exceeds 8e-3.  The background
  log-odds log(bg / (1 - bg)), bg = prod_k (1 - p_k), move by -sum_k p_k dl_k / (1 - bg), and the engine's object-logit
  errors dl_k are mostly a bias of one sign, common to every object (the 'mean error' rows; fp16 weight rounding, which
  every object shares, is the likely source), so where all 16 objects claim a pixel they add up.  The row is kept at its bound and the case is reported as an expected failure while it is the only
  failing row; any other failure fails the case, and the case fails too once the row meets its bound again.

The exact properties at the end pin what the engine's results must not depend on: how the objects are chunked, whether
the sensory state is updated, and which other objects share the batch.
"""
import math
import os
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import network as onet

pytestmark = pytest.mark.gpu

CASES = {  # name: (frame size before padding, objects, decode steps)
    'c2': ((480, 854), 5, 3),
    'c3': ((1080, 1920), 16, 2),
}
# test_stages_gpu.py's per-stage bounds: (kind, bound), kind 'rel' = max abs error / max |float64|
BOUNDS = {
    'features': ('rel', 8e-4),
    'key': ('abs', 3e-4), 'shrinkage': ('abs', 3e-4), 'selection': ('abs', 5e-5),
    'value': ('rel', 2.5e-3),
    'sensory (encode)': ('abs', 8e-3),
    'sensory (decode)': ('abs', 2e-2),
    'logits': ('abs', 8e-3),
    'prob': ('abs', 1e-3),
}
# regression ceilings: the largest error measured at each case (H100 80GB HBM3) plus about 10 %
CEILINGS = {
    'c2': {'logits': ('abs', 3.1e-3), 'prob': ('abs', 4.5e-4)},  # measured 2.78e-3, 4.03e-4
    'c3': {'logits': ('abs', 3.0e-3), 'prob': ('abs', 1.3e-4)},  # measured 2.75e-3, 1.17e-4
}
KNOWN_MISSES = {  # (case, stage): why the row misses its bound
    ('c3', 'logits (agg. background)'):
        'the background log-odds sum the 16 objects\' same-signed logit errors (measured 1.4e-2 / 1.5e-2 at frames 1 / 2)',
}


# ------------------------------------------------------------------------------------------------------- inputs
def _frames(golden_dir, hw, n):
    """The first n config-1 frames at size hw, ImageNet-normalised and padded: fp32 [n,3,H,W] on the device."""
    from deva.inference.frame_io import IMAGENET_MEAN, IMAGENET_STD
    from deva.utils.tensor_utils import pad_divide_by
    u8 = np.load(os.path.join(golden_dir, 'config1_vos.npz'))['frames_u8'][:n]
    x = torch.from_numpy(u8).cuda().permute(0, 3, 1, 2).float() / 255
    if tuple(x.shape[-2:]) != hw:
        x = F.interpolate(x, size=hw, mode='bilinear', align_corners=False)
    mean = torch.tensor(IMAGENET_MEAN, device='cuda').view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD, device='cuda').view(1, 3, 1, 1)
    x, _ = pad_divide_by((x - mean) / std, 16)
    return x.contiguous()


def _soft_masks(k, hw):
    """k overlapping ellipses with sigmoid edges a few pixels wide, scaled where they overlap so that they sum to at
    most 1 (to fp32 rounding), padded like the frames: fp32 [1,k,H,W] on the device."""
    from deva.utils.tensor_utils import pad_divide_by
    h, w = hw
    yy = torch.arange(h, dtype=torch.float64, device='cuda').view(-1, 1) + 0.5
    xx = torch.arange(w, dtype=torch.float64, device='cuda').view(1, -1) + 0.5
    edge = h / 120
    planes = []
    for i in range(k):
        t = 2 * math.pi * i / k
        cy, cx = h * (0.5 + 0.27 * math.sin(t + 0.4)), w * (0.5 + 0.3 * math.cos(t))
        a, b = w * (0.09 + 0.04 * (i % 3)), h * (0.12 + 0.05 * (2 * i % 3))
        c, s = math.cos(0.6 * i), math.sin(0.6 * i)
        u, v = ((xx - cx) * c + (yy - cy) * s) / a, ((yy - cy) * c - (xx - cx) * s) / b
        planes.append(torch.sigmoid((1 - torch.sqrt(u * u + v * v)) * min(a, b) / edge))
    m = torch.stack(planes)
    m = m / m.sum(0).clamp_min(1)
    m, _ = pad_divide_by(m.float().unsqueeze(0), 16)
    return m.contiguous()


@pytest.fixture(scope='module')
def engine(synthetic_sd):
    from deva.model.native_engine import NativeEngine
    from deva import _native
    _native.require_device()
    return NativeEngine({k: v.cuda() for k, v in synthetic_sd.items()})


@pytest.fixture(scope='module')
def sd64(synthetic_sd):
    return {k: (v.double() if v.is_floating_point() else v).cuda() for k, v in synthetic_sd.items()}


# ------------------------------------------------------------------------------------------------------- float64 side
def _oracle_encode_mask(sd, image, ms, sensory, masks):
    outs = [onet.encode_mask(sd, image, ms, sensory[:, i:i + 1], masks[:, i:i + 1]) for i in range(masks.shape[1])]
    return torch.cat([v for v, _ in outs], 1), torch.cat([s for _, s in outs], 1)


def _oracle_decode(sd, ms, readout, sensory, masks):
    outs = [onet.decode(sd, ms, readout[:, i:i + 1], sensory[:, i:i + 1], masks[:, i:i + 1])
            for i in range(masks.shape[1])]
    return torch.cat([s for s, _ in outs], 1), torch.cat([lg for _, lg in outs], 1)


class Table:
    """Measured errors beside their bounds; every row is printed before any bound is asserted."""

    def __init__(self, case, known_misses=None):
        self.case, self.rows = case, []
        self.known_misses = KNOWN_MISSES if known_misses is None else known_misses

    def add(self, step, stage, got, want, bound_key=None, bound=None):
        """max |got - want| (over max |want| for a 'rel' bound) against BOUNDS[bound_key or stage], or `bound`."""
        kind, limit = bound or BOUNDS[bound_key or stage]
        assert tuple(got.shape) == tuple(want.shape), (stage, got.shape, want.shape)
        err = float((got.double() - want).abs().max())
        if kind == 'rel':
            err /= max(float(want.abs().max()), 1e-30)
        self.rows.append((step, stage, kind, err, limit, bool(err < limit)))  # NaN fails

    def note(self, step, stage, value):
        """A measured value printed for context, with no bound."""
        self.rows.append((step, stage, '', value, None, True))

    def report(self, seconds, peak_gib):
        print(f'\n{self.case}: float64 engine check, {seconds:.1f} s, peak device memory {peak_gib:.2f} GiB')
        for step, stage, kind, err, limit, ok in self.rows:
            tail = '' if limit is None else f'  bound {limit:.1e}  {"ok" if ok else "FAIL"}'
            print(f'    {step:8s} {stage:30s} {kind:4s} {err:+.3e}{tail}')
        bad = [r for r in self.rows if not r[-1]]
        unexpected = [r for r in bad if (self.case, r[1]) not in self.known_misses]
        assert not unexpected, unexpected
        known = [stage for case, stage in self.known_misses if case == self.case]
        met = [s for s in known if not any(r[1] == s for r in bad)]
        assert not met, f'{met} now meet their bounds at {self.case}: take them out of KNOWN_MISSES'
        if bad:
            pytest.xfail('; '.join(f'{s}: {self.known_misses[(self.case, s)]}' for s in known))


@pytest.mark.parametrize('case', list(CASES))
def test_engine_matches_float64(case, engine, sd64, golden_dir):
    hw, k, steps = CASES[case]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    tab = Table(case)
    compare_with_float64(engine, sd64, _frames(golden_dir, hw, steps + 1), _soft_masks(k, hw), tab, CEILINGS[case])
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() / 2**30
    torch.cuda.empty_cache()
    tab.report(seconds, peak)


def compare_with_float64(engine, sd64, frames, masks, tab, ceilings=None):
    """Frame 0 through both encoders and the value encoder, then one decode per further frame, each side carrying its
    own features and sensory state, every stage's error added to ``tab`` (and the regression ceilings, when given)."""
    steps, k = frames.shape[0] - 1, masks.shape[1]
    masks64 = masks.double()

    def features(t):
        image = frames[t:t + 1]
        ms, feat = engine.encode_image(image)
        ms64, feat64 = onet.encode_image(sd64, image.double())
        step = f'frame {t}'
        for name, got, want in zip(('f16', 'f8', 'f4'), ms, ms64):
            tab.add(step, name, got, want, 'features')
        if t == 0:
            tab.add(step, 'key_feat', feat, feat64, 'features')
            for name, got, want in zip(('key', 'shrinkage', 'selection'), engine.transform_key(feat),
                                       onet.transform_key(sd64, feat64)):
                tab.add(step, name, got, want)
        return image, ms, ms64

    # frame 0: both encoders, the value encoder from a zero sensory state
    image, ms, ms64 = features(0)
    hh, ww = ms[0].shape[-2:]
    zero = torch.zeros(1, k, engine.value_dim, hh, ww, dtype=torch.float16, device='cuda')
    value, sensory = engine.encode_mask(image, ms, zero, masks)
    value64, sensory64 = _oracle_encode_mask(sd64, image.double(), ms64, zero.double(), masks64)
    tab.add('frame 0', 'value', value, value64)
    tab.add('frame 0', 'sensory', sensory, sensory64, 'sensory (encode)')
    readout = value64.half()  # the memory readout both sides decode from
    readout64 = readout.double()
    del value, value64, zero

    # frames 1..n: each side decodes from its own features and carries its own sensory state
    for t in range(1, steps + 1):
        _, ms, ms64 = features(t)
        sensory, logits = engine.decode(ms, readout, sensory, masks)
        sensory64, logits64 = _oracle_decode(sd64, ms64, readout64, sensory64, masks64)
        step = f'frame {t}'
        tab.add(step, 'logits (object)', logits, logits64, 'logits')
        if ceilings:
            tab.add(step, '  regression ceiling (logits)', logits, logits64, bound=ceilings['logits'])
        tab.note(step, '  mean error (bias)', float((logits.double() - logits64).mean()))
        tab.add(step, 'sensory', sensory, sensory64, 'sensory (decode)')
        full, prob = engine.probabilities(logits.float().contiguous(), want_logits=True)
        full64, prob64 = onet.output_tail(logits64)
        # the bound of test_stages_gpu.py on every channel, the object channels and the background reported apart
        tab.add(step, 'logits (agg. objects)', full[:, 1:], full64[:, 1:], 'logits')
        tab.add(step, 'logits (agg. background)', full[:, :1], full64[:, :1], 'logits')
        tab.add(step, 'prob', prob, prob64)
        # the engine's own logits through the float64 tail: what the logit errors alone do to the rows above
        full_x, prob_x = onet.output_tail(logits.double())
        tab.note(step, '  float64 tail: agg. background', float((full_x[:, :1] - full64[:, :1]).abs().max()))
        tab.note(step, '  float64 tail: prob', float((prob_x - prob64).abs().max()))
        del full_x, prob_x
        if ceilings:
            tab.add(step, '  regression ceiling (prob)', prob, prob64, bound=ceilings['prob'])
        del ms, ms64, logits, logits64, full, full64, prob, prob64


# ------------------------------------------------------------------------------------------------------- exact properties
def _bits(t):
    t = t.contiguous()
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _same_bits(a, b):
    return a.dtype == b.dtype and tuple(a.shape) == tuple(b.shape) and torch.equal(_bits(a), _bits(b))


@pytest.fixture(scope='module')
def c3_native(engine, golden_dir):
    """c3's shape (1088 x 1920, 16 objects), native only: frame 0 encoded into (value, sensory) from a zero state and
    frame 1's features as the inputs, and the reference results of the 16-object batch run once on those inputs:
    encode_mask (frame 0, from that sensory) -> enc, decode (frame 1) -> dec."""
    hw, k, _ = CASES['c3']
    frames = _frames(golden_dir, hw, 2)
    masks = _soft_masks(k, hw)
    image = frames[0:1]
    ms0, _ = engine.encode_image(image)
    ms1, _ = engine.encode_image(frames[1:2])
    hh, ww = ms0[0].shape[-2:]
    zero = torch.zeros(1, k, engine.value_dim, hh, ww, dtype=torch.float16, device='cuda')
    value, sensory = engine.encode_mask(image, ms0, zero, masks)
    enc = engine.encode_mask(image, ms0, sensory, masks)
    dec = engine.decode(ms1, value, sensory, masks)
    yield dict(image=image, ms0=ms0, ms1=ms1, masks=masks, value=value, sensory=sensory, enc=enc, dec=dec)
    torch.cuda.empty_cache()


def test_chunked_objects_are_bit_identical(engine, c3_native):
    """chunk_size=5 (chunks of 5, 5, 5, 1 objects) against all 16 in one batch."""
    s = c3_native
    (value, sensory), (sensory_d, logits) = s['enc'], s['dec']
    value5, sensory5 = engine.encode_mask(s['image'], s['ms0'], s['sensory'], s['masks'], chunk_size=5)
    assert _same_bits(value5, value), 'encode_mask value'
    assert _same_bits(sensory5, sensory), 'encode_mask sensory'
    sensory5, logits5 = engine.decode(s['ms1'], s['value'], s['sensory'], s['masks'], chunk_size=5)
    assert _same_bits(sensory5, sensory_d), 'decode sensory'
    assert _same_bits(logits5, logits), 'decode logits'


def test_paths_without_a_sensory_update_are_bit_identical(engine, c3_native):
    """decode(update_sensory=False) asks the logit head's conv for no 4x4 pool (its tile may differ) and
    encode_mask(deep_update=False) skips the GRU: the results they do produce are the same bits, and the sensory state
    comes back as the very object that went in."""
    s = c3_native
    kept, logits_nu = engine.decode(s['ms1'], s['value'], s['sensory'], s['masks'], update_sensory=False)
    assert kept is s['sensory']
    assert _same_bits(logits_nu, s['dec'][1])
    value_nu, kept = engine.encode_mask(s['image'], s['ms0'], s['sensory'], s['masks'], deep_update=False)
    assert kept is s['sensory']
    assert _same_bits(value_nu, s['enc'][0])


@pytest.mark.parametrize('obj', [0, 7, 15])
def test_object_alone_equals_its_row_of_the_batch(engine, c3_native, obj):
    """One object run alone (K = 1: the fusers' shared half is an ordinary residual) gives the bits of its row of the
    16-object run (the shared half broadcast across the batch)."""
    s = c3_native
    one = slice(obj, obj + 1)
    (value, sensory), (sensory_d, logits) = s['enc'], s['dec']
    value1, sensory1 = engine.encode_mask(s['image'], s['ms0'], s['sensory'][:, one], s['masks'][:, one])
    assert _same_bits(value1, value[:, one]), 'encode_mask value'
    assert _same_bits(sensory1, sensory[:, one]), 'encode_mask sensory'
    sensory1, logits1 = engine.decode(s['ms1'], s['value'][:, one], s['sensory'][:, one], s['masks'][:, one])
    assert _same_bits(sensory1, sensory_d[:, one]), 'decode sensory'
    assert _same_bits(logits1, logits[:, one]), 'decode logits'
