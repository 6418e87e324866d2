"""The native engine and each of its convolution launches against float64, at the frame sizes and object counts real
videos reach beyond the benchmark's c2 (480p, 5 objects) and c3 (1080p, 16 objects).

The kernels are swept on their own (tests/golden/conv_cases.py), but the host picks each launch's schedule from the
frame size and the object count K: ``native_ops.choose_tile`` the pixel tile from the output sides, ``choose_nt`` the
channel tile from ``b * pixel_tiles`` against the SM count (b = K for per-object layers), ``encode_mask`` / ``decode``
the object chunks, ``output_tail`` its register path (K + 1 <= 32) or the one that stashes logits in ``prob``, and
``stem_im2col`` one of three kernels with row and column tails that depend on the frame size.  The cases below come
from the drivers' own size rule (``frame_io.reader_size``, padded to 16), with no resize for ``--size -1``:

    single    480 x 854 at 480, K = 1          a DAVIS video with one object
    portrait  1280 x 720 at 480, K = 3         a portrait YouTube-VOS clip (864 x 480 padded)
    ms240 / ms360 / ms600  720 x 1280, K = 2 / 2 / 5   multi-scale members: 1/16 sides 15 x 27, 23 x 40, 38 x 67
    many      480 x 854 at 480, K = 33         a detection session with more objects than the output tail's registers
    many/8    the same with chunk_size = 8     chunks of 8, 8, 8, 8 and 1 objects (per-launch check)
    small     100 x 150, size -1, K = 1        1/16 is 7 x 10
    4k        2160 x 3840, size -1, K = 1      1/16 is 135 x 240 (per-launch check only)

At every case each ``conv2d`` launch of encode_image, transform_key, encode_mask and one decode with the sensory update
is checked against oracle/conv_desc.py with the (4 n_k + 8) 2^-23 M bound of test_conv_engine_launches_gpu.py, and
(except at 4k and many/8) the whole engine against the float64 oracle network with the bounds of
test_engine_float64_gpu.py.  At ``many`` the chunked run must equal the unchunked one bit for bit, and an object run
alone its row of the batch.

The coverage test records the launch descriptors of every case and of c2 and c3 and fails when the new cases stop
reaching a tall rectangle (th > tw), flat tiles on an odd 1/16 side, chunked per-object launches in encode_mask and
decode, the output tail at K + 1 > 32, or the pixel-per-thread stem_im2col forms at a width whose half is not a
multiple of 128.  It prints the (tile, channel tile, k-split, epilogue, mode) combinations c2 and c3 never reach.

``conv_ex`` splits a precise layer's chain into split-K parts plus ``sum_parts`` only when the residual is not
broadcast (``res is None or res.shape[0] == b``), so a precise layer whose residual is shared across objects would take
that path at K = 1 only.  Reading the engine: the precise layers with a residual are the pixel encoder's ``c3``
(batch 1, 3 to 12 k-iterations) and the fusers' ``b1.ds_g`` (broadcast at K > 1; a 1x1 over 256 or 512 channels in
three passes, 12 or 24 k-iterations).  None is longer than ``MAX_CHAIN`` (32), so no residual ever reaches
``sum_parts`` at any K: the automatic split-K path is taken only by residual-free layers of the pixel encoder (the 3x3
``c2`` of layer2 and layer3, the 1x1 ``c1`` over 1024 channels of layer3.1-5, and proj1 / proj2).  The coverage test lists those layers and fails if a ``sum_parts`` call ever carries a
residual, since that path would then need a case of its own here.

Two rows miss their bounds for reasons measured and written down in KNOWN_MISSES; each case is reported as an
expected failure while its row is the only one failing.  Both are the engine's object-logit error (within 2.4e-3 / 3e-3
of float64, against a bound of 8e-3, with a bias of one sign: the 'mean error' rows) carried through the output tail,
which itself adds nothing: the engine's own logits through the float64 tail (the 'float64 tail' rows) reproduce both
misses to three digits.  At K = 1 the softmax over (background, object) = (-l, l) is sigmoid(2 l), twice as steep as
a single object's probability, so ``single``'s prob exceeds 1e-3 by 5 % at one frame.  At K = 33 the background
log-odds add up the objects' same-signed errors, as at c3.

Finally the three ``stem_im2col`` kernels (pixel-per-thread C = 1 / C = 3 with and without the fp16 remainder, and the
generic shared-memory kernel, which C = 1 with a remainder and any other C <= 8 reach) and ``nchw_to_nhwc`` are checked
bit for bit against float64 ``F.unfold`` / a permute, into NaN-filled buffers with guard regions.
"""
import os
import sys
import time

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_conv_engine_launches_gpu as tcl  # noqa: E402  (the per-launch Recorder and its bound)
import test_engine_float64_gpu as tef  # noqa: E402  (inputs, bounds and the float64 comparison)
import test_network_helpers_gpu as tnh  # noqa: E402  (NaN-filled outputs with guard regions)

from deva.inference.frame_io import reader_size  # noqa: E402

gpu = pytest.mark.gpu
needs_device = pytest.mark.skipif(not torch.cuda.is_available(), reason='needs a CUDA device')


# ------------------------------------------------------------------------------------------------------- cases
def working_size(src, size):
    """The frame size the drivers feed the network: ``reader_size`` of the source at ``size`` (none for size -1)."""
    return reader_size(*src, size) if size > 0 else tuple(src)


def padded(hw):
    return tuple(-(-s // 16) * 16 for s in hw)


# name: (source h x w, size, objects, decode steps of the float64 check (0: none), chunk_size)
CASES = {
    'single': ((480, 854), 480, 1, 3, -1),
    'portrait': ((1280, 720), 480, 3, 3, -1),
    'ms240': ((720, 1280), 240, 2, 3, -1),
    'ms360': ((720, 1280), 360, 2, 3, -1),
    'ms600': ((720, 1280), 600, 5, 3, -1),
    'many': ((480, 854), 480, 33, 3, -1),
    'many/8': ((480, 854), 480, 33, 0, 8),
    'small': ((100, 150), -1, 1, 3, -1),
    '4k': ((2160, 3840), -1, 1, 0, -1),
}
F64_CASES = [c for c in CASES if CASES[c][3]]
KNOWN_MISSES = {  # (case, stage): why the row misses its bound (H100 80GB HBM3), as test_engine_float64_gpu.py's
    ('single', 'prob'):
        'with one object prob = sigmoid(2 l) of the object logit l, so a logit error dl moves prob by up to dl / 2 at '
        'the mask edge: object logits within 2.4e-3 of float64 (bound 8e-3) put prob 1.05e-3 off at frame 2 '
        '(7.1e-4 / 8.5e-4 at frames 1 / 3), and the engine\'s logits through the float64 tail give the same 1.05e-3',
    ('many', 'logits (agg. background)'):
        'as at c3, the background log-odds sum the 33 objects\' same-signed logit errors (measured 1.13e-2 / 1.62e-2 / '
        '9.5e-3 at frames 1 / 2 / 3, the same through the float64 tail); prob stays within 5.1e-5',
}


def _case(name):
    src, size, k, steps, chunk = CASES[name]
    return working_size(src, size), k, steps, chunk


def test_case_table_reaches_the_sides_it_is_for():
    """The 1/16 sides each case stands for follow from the drivers' size rule."""
    sides = {name: tuple(s // 16 for s in padded(_case(name)[0])) for name in CASES}
    assert sides['single'] == sides['many'] == (30, 54)  # c2's
    assert sides['portrait'] == (54, 30)
    assert (sides['ms240'], sides['ms360'], sides['ms600']) == ((15, 27), (23, 40), (38, 67))
    assert sides['small'] == (7, 10) and sides['4k'] == (135, 240)


# ------------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope='module', autouse=True)
def _duration():
    t0 = time.perf_counter()
    yield
    print(f'\ntest_engine_shapes_gpu.py: {time.perf_counter() - t0:.1f} s')


@pytest.fixture(scope='module')
def engine(synthetic_sd):
    from deva.model.native_engine import NativeEngine
    from deva import _native
    _native.require_device()
    return NativeEngine({k: v.cuda() for k, v in synthetic_sd.items()})


@pytest.fixture(scope='module')
def sd64(synthetic_sd):
    return {k: (v.double() if v.is_floating_point() else v).cuda() for k, v in synthetic_sd.items()}


# ------------------------------------------------------------------------------------------------------- per launch
@gpu
@needs_device
@pytest.mark.parametrize('case', list(CASES))
def test_every_launch_within_its_bound(case, engine, golden_dir, monkeypatch):
    from deva import _native as nat
    t0 = time.perf_counter()
    hw, k, _, chunk = _case(case)
    frames = tef._frames(golden_dir, hw, 2)
    masks = tef._soft_masks(k, hw)
    rec = tcl.Recorder(engine, nat.conv2d)
    monkeypatch.setattr(nat, 'conv2d', rec)
    tcl.run_stages(engine, rec, frames, masks, chunk_size=chunk)
    monkeypatch.undo()
    torch.cuda.synchronize()
    del frames, masks
    torch.cuda.empty_cache()
    tcl.report(f'{case} ({hw[0]} x {hw[1]}, K = {k}, chunk_size {chunk})', rec.rows, time.perf_counter() - t0)


# ------------------------------------------------------------------------------------------------------- float64
@gpu
@needs_device
@pytest.mark.parametrize('case', F64_CASES)
def test_engine_matches_float64(case, engine, sd64, golden_dir):
    hw, k, steps, _ = _case(case)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    tab = tef.Table(case, KNOWN_MISSES)
    tef.compare_with_float64(engine, sd64, tef._frames(golden_dir, hw, steps + 1), tef._soft_masks(k, hw), tab)
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() / 2**30
    torch.cuda.empty_cache()
    tab.report(seconds, peak)


@pytest.fixture(scope='module')
def many_native(engine, golden_dir):
    """``many``'s shape (480 x 864, 33 objects), native only, as test_engine_float64_gpu.py's c3_native: frame 0 encoded
    from a zero state, frame 1's features, and the 33-object batch's encode_mask -> enc and decode -> dec."""
    hw, k, _, _ = _case('many')
    frames = tef._frames(golden_dir, hw, 2)
    masks = tef._soft_masks(k, hw)
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


@gpu
@needs_device
def test_many_chunked_objects_are_bit_identical(engine, many_native):
    """chunk_size=8 (chunks of 8, 8, 8, 8, 1 objects) against all 33 in one batch, and the output tail of both."""
    s = many_native
    (value, sensory), (sensory_d, logits) = s['enc'], s['dec']
    value8, sensory8 = engine.encode_mask(s['image'], s['ms0'], s['sensory'], s['masks'], chunk_size=8)
    assert tef._same_bits(value8, value), 'encode_mask value'
    assert tef._same_bits(sensory8, sensory), 'encode_mask sensory'
    sensory8, logits8 = engine.decode(s['ms1'], s['value'], s['sensory'], s['masks'], chunk_size=8)
    assert tef._same_bits(sensory8, sensory_d), 'decode sensory'
    assert tef._same_bits(logits8, logits), 'decode logits'
    full8, prob8 = engine.probabilities(logits8.float().contiguous(), want_logits=True)
    full, prob = engine.probabilities(logits.float().contiguous(), want_logits=True)
    assert tef._same_bits(full8, full) and tef._same_bits(prob8, prob), 'output tail'


@gpu
@needs_device
@pytest.mark.parametrize('obj', [0, 16, 32])
def test_many_object_alone_equals_its_row_of_the_batch(engine, many_native, obj):
    """One object run alone (K = 1) gives the bits of its row of the 33-object run."""
    s = many_native
    one = slice(obj, obj + 1)
    (value, sensory), (sensory_d, logits) = s['enc'], s['dec']
    value1, sensory1 = engine.encode_mask(s['image'], s['ms0'], s['sensory'][:, one], s['masks'][:, one])
    assert tef._same_bits(value1, value[:, one]), 'encode_mask value'
    assert tef._same_bits(sensory1, sensory[:, one]), 'encode_mask sensory'
    sensory1, logits1 = engine.decode(s['ms1'], s['value'][:, one], s['sensory'][:, one], s['masks'][:, one])
    assert tef._same_bits(sensory1, sensory_d[:, one]), 'decode sensory'
    assert tef._same_bits(logits1, logits[:, one]), 'decode logits'


# ------------------------------------------------------------------------------------------------------- coverage
def _record(engine, golden_dir, monkeypatch, hw, k, chunk):
    """Launch descriptors (Recorder rows, no oracle) of run_stages plus the output tail, and the calls of sum_parts,
    stem_im2col and output_tail as (function, stage, preceding conv layer, arguments)."""
    from deva import _native as nat
    frames = tef._frames(golden_dir, hw, 2)
    masks = tef._soft_masks(k, hw)
    rec = tcl.Recorder(engine, nat.conv2d, check=False)
    calls = []

    def spy(name):
        real = getattr(nat, name)

        def call(*args, **kwargs):
            calls.append((name, rec.stage, rec.rows[-1]['layer'] if rec.rows else '', args, kwargs))
            return real(*args, **kwargs)
        return call
    monkeypatch.setattr(nat, 'conv2d', rec)
    for name in ('sum_parts', 'stem_im2col', 'output_tail'):
        monkeypatch.setattr(nat, name, spy(name))
    _, logits = tcl.run_stages(engine, rec, frames, masks, chunk_size=chunk)
    rec.stage = 'output_tail'
    engine.probabilities(logits.float().contiguous(), want_logits=True)
    monkeypatch.undo()
    torch.cuda.synchronize()
    return rec.rows, calls


def _combo(r):
    return (r['tile'], r['nt'], r['ksplit'], r['epi'], r['mode'])


@gpu
@needs_device
def test_new_cases_reach_what_c2_and_c3_do_not(engine, golden_dir, monkeypatch):
    t0 = time.perf_counter()
    seen = {}
    for name, (hw, k, _) in tef.CASES.items():
        seen[name] = (padded(hw), k) + _record(engine, golden_dir, monkeypatch, hw, k, -1)
    for name in CASES:
        hw, k, _, chunk = _case(name)
        seen[name] = (padded(hw), k) + _record(engine, golden_dir, monkeypatch, hw, k, chunk)
    new = list(CASES)

    def out_hw(r):
        h, w = (int(s) for s in r['shape'].split('x')[1:])
        return engine.P[r['layer']].out_hw(h, w)

    def per_object(r, stage, b):
        return r['stage'] == stage and r['shape'].startswith(f'{b}x') and r['layer'].split('.')[1] in (
            'stem_mask', 'layer1', 'layer2', 'layer3', 'gru', 'sensory_compress', 'up_16_8', 'up_8_4', 'su')

    reached = {
        'a tall rectangle (th > tw)': [
            n for n in new if any(r['tile'] != 'flat' and int(r['tile'].split('x')[0]) > int(r['tile'].split('x')[1])
                                  for r in seen[n][2])],
        'flat tiles on an odd 1/16 side': [
            n for n in new if any(r['tile'] == 'flat' and out_hw(r) == tuple(s // 16 for s in seen[n][0])
                                  and (out_hw(r)[0] % 2 or out_hw(r)[1] % 2) for r in seen[n][2])],
        'chunked encode_mask and decode': [
            n for n in new if all(any(per_object(r, st, b) for r in seen[n][2])
                                  for st in ('encode_mask', 'decode') for b in (8, 1)) and seen[n][1] > 8],
        'the output tail at K + 1 > 32': [
            n for n in new if any(c[0] == 'output_tail' and c[3][4] + 1 > 32 for c in seen[n][3])],
    }
    for c, kp, lo in ((1, 64, False), (3, 192, False), (3, 192, True)):
        reached[f'the pixel-per-thread stem_im2col C = {c}{" with dst_lo" if lo else ""} at W/2 % 128 != 0'] = [
            n for n in new if any(f == 'stem_im2col' and a[3] == c and a[6] == kp and (kw.get('dst_lo') is not None) == lo
                                  and (a[5] // 2) % 128 for f, _, _, a, kw in seen[n][3])]
    print(f'\ncoverage of the new cases ({time.perf_counter() - t0:.1f} s to record {len(seen)} cases):')
    for what, names in reached.items():
        print(f'    {what:60s} {", ".join(names) if names else "NOT REACHED"}')

    # the automatic split-K path: its conv launches, and whether sum_parts got a residual
    print('    automatic split-K (conv_ex -> sum_parts), by case: layer [residual]')
    with_res = []
    for n, (_, k, _, calls) in seen.items():
        auto = [(c[2], c[4].get('res') is not None) for c in calls if c[0] == 'sum_parts']
        with_res += [(n, layer) for layer, res in auto if res]
        print(f'      {n:9s} K={k:2d}: ' + ', '.join(sorted({f'{layer}{" [res]" if res else ""}' for layer, res in auto})))

    base = {_combo(r) for n in tef.CASES for r in seen[n][2]}
    fresh = {}
    for n in new:
        for r in seen[n][2]:
            if _combo(r) not in base:
                fresh.setdefault(_combo(r), []).append(n)
    print(f'    {len(fresh)} (tile, nt, ksplit, epilogue, mode) combinations c2 and c3 never reach:')
    for combo in sorted(fresh, key=str):
        tile, nt, ks, epi, mode = combo
        print(f'      {tile:6s} {nt:4d} {ks:2d} {epi:6s} {mode:24s} {", ".join(sorted(set(fresh[combo])))}')
    missing = [what for what, names in reached.items() if not names]
    assert not missing, f'the new cases no longer reach {missing}'
    assert not with_res, (f'sum_parts now adds a residual at {with_res}: the split-K path with a residual needs a case '
                          'of its own (see the module docstring)')


# ------------------------------------------------------------------------------------------------------- stem_im2col
def stem_columns_ref(planes, k_pad):
    """The 7x7 stride-2 pad-3 im2col of float planes [B, C, H, W] as [B, H/2, W/2, k_pad], column (kh * 7 + kw) * C + c
    and zeros past 49 C: ``F.unfold`` (columns c * 49 + kh * 7 + kw) rearranged."""
    b, c, h, w = planes.shape
    cols = F.unfold(planes, 7, padding=3, stride=2)  # [B, C*49, L]
    cols = cols.view(b, c, 49, -1).permute(0, 3, 2, 1).reshape(b, h // 2, w // 2, 49 * c)
    return F.pad(cols, (0, k_pad - 49 * c))


def _stem_columns_loop(planes, k_pad):
    b, c, h, w = planes.shape
    out = torch.zeros(b, h // 2, w // 2, k_pad, dtype=planes.dtype)
    for i in range(b):
        for yo in range(h // 2):
            for xo in range(w // 2):
                for ky in range(7):
                    for kx in range(7):
                        y, x = 2 * yo - 3 + ky, 2 * xo - 3 + kx
                        if 0 <= y < h and 0 <= x < w:
                            for ch in range(c):
                                out[i, yo, xo, (ky * 7 + kx) * c + ch] = planes[i, ch, y, x]
    return out


def _split16(v64):
    """hi = fp16(v) round to nearest, lo = fp16(v - hi): v - hi is exact for fp32 v, so one rounding each."""
    hi = v64.half()
    return hi, (v64 - hi.double()).half()


@pytest.mark.parametrize('b, c, h, w', [(1, 1, 2, 2), (2, 2, 6, 10), (1, 3, 8, 4), (2, 5, 4, 14)])
def test_stem_columns_ref_matches_a_direct_loop(b, c, h, w):
    g = torch.Generator().manual_seed(b * 100 + c * 10 + h + w)
    planes = torch.randn(b, c, h, w, generator=g, dtype=torch.float64)
    k_pad = -(-49 * c // 64) * 64
    assert torch.equal(stem_columns_ref(planes, k_pad), _stem_columns_loop(planes, k_pad))


def _planes(b, c, h, w, seed):
    """fp32 planes of normal values, a tenth of them scaled down to fp16-subnormal size, where hi and lo round coarsely."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(b, c, h, w, device='cuda', generator=g) * 3
    tiny = torch.rand(b, c, h, w, device='cuda', generator=g) < 0.1
    return torch.where(tiny, x * 2.0 ** -18, x).contiguous()


STEM_FORMS = [  # (C, Kp, with dst_lo): which kernel csrc/elementwise.cu deva_b200_stem_im2col launches
    (1, 64, False),   # pixel-per-thread, 4 rows per block (the mask stem)
    (3, 192, False),  # pixel-per-thread, 2 rows per block (the mask encoder's image stem)
    (3, 192, True),   # the same with the fp16 remainder (the pixel encoder's stem)
    (1, 64, True),    # generic: C = 1 with a remainder has no pixel-per-thread form
    (2, 128, False), (2, 128, True), (5, 256, False), (5, 256, True),  # generic
]
# (b, h, w): W/2 = 300 and 129 are multiples of neither 128 nor 64, H/2 = 7 and 9 are odd (the row tails of both
# pixel-per-thread forms), and a 2 x 2 input is one output pixel whose taps are mostly padding
STEM_SHAPES = [(2, 14, 600), (3, 18, 258), (1, 2, 2)]


@gpu
@needs_device
@pytest.mark.parametrize('b, h, w', STEM_SHAPES)
@pytest.mark.parametrize('c, k_pad, with_lo', STEM_FORMS)
def test_stem_im2col_bit_exact(c, k_pad, with_lo, b, h, w):
    nat = tnh._nat()
    planes = _planes(b, c, h, w, seed=c * 1000 + h * 10 + w)
    outs = tnh.Outputs()
    hi = outs.new((b, h // 2, w // 2, k_pad), torch.float16)
    lo = outs.new((b, h // 2, w // 2, k_pad), torch.float16) if with_lo else None
    nat.stem_im2col(planes, hi, b, c, h, w, k_pad, dst_lo=lo)
    torch.cuda.synchronize()
    outs.check()
    want_hi, want_lo = _split16(stem_columns_ref(planes.double(), k_pad))
    bad = (hi.view(torch.int16) != want_hi.view(torch.int16)).nonzero()
    assert bad.shape[0] == 0, f'hi differs at {bad.shape[0]} elements, first [b, y, x, column] {bad[0].tolist()}'
    if with_lo:
        bad = (lo.view(torch.int16) != want_lo.view(torch.int16)).nonzero()
        assert bad.shape[0] == 0, f'lo differs at {bad.shape[0]} elements, first [b, y, x, column] {bad[0].tolist()}'


@gpu
@needs_device
@pytest.mark.parametrize('b, c, h, w, c_pad', [(2, 3, 7, 9, 8), (1, 5, 13, 17, 64), (3, 1, 1, 1, 8), (1, 3, 11, 5, 3),
                                               (2, 64, 5, 3, 64)])
def test_nchw_to_nhwc_bit_exact(b, c, h, w, c_pad):
    nat = tnh._nat()
    src = _planes(b, c, h, w, seed=b + c + h + w + c_pad)
    outs = tnh.Outputs()
    dst = outs.new((b, h, w, c_pad), torch.float16)
    nat.nchw_to_nhwc(src, dst, b, c, h, w, c_pad)
    torch.cuda.synchronize()
    outs.check()
    want = F.pad(src.double().permute(0, 2, 3, 1), (0, c_pad - c)).half()
    assert torch.equal(dst.view(torch.int16), want.view(torch.int16))
