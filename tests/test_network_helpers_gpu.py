"""The network path's helper kernels (csrc/elementwise.cu) against float64 references at the shapes the network runs.

Every output is written into a view of a larger NaN-filled buffer with a guard region behind it: a test fails when an
output element is left unwritten or a kernel writes past its output.  References are built in float64 from the exact
inputs (a split pair (hi, lo) stands for hi + lo) and reuse oracle/network.py where it states the operation.  Kernels
whose arithmetic is fixed - a fixed-order fp32 sum, a max, a round-to-nearest hi/lo split - are also compared bit for
bit with the same fp32 operations done in torch.  Each test prints its measured error beside its bound.

Network shapes: 480p pads to 480 x 864 (f4 = 120 x 216, f8 = 60 x 108, f16 = 30 x 54), 1080p to 1088 x 1920
(f16 = 68 x 120); K is the number of objects.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import network as onet

GUARD = 64
U8_FILL = 0xFF     # an e4m3 NaN: the satfinite conversion never produces it
EPS32 = 2.0 ** -23
KS = (1, 5, 16)


def _nat():
    from deva import _native
    _native.require_device()
    return _native


# ------------------------------------------------------------------------------------------------- output placement
class Outputs:
    """Output tensors as views of larger buffers filled with NaN (0xFF for bytes), each followed by a guard region."""

    def __init__(self, device='cuda'):
        self.device = device
        self.bufs = []

    def new(self, shape, dtype):
        n = math.prod(shape)
        buf = torch.empty(n + GUARD, dtype=dtype, device=self.device)
        buf.fill_(U8_FILL if dtype == torch.uint8 else float('nan'))
        self.bufs.append((buf, n))
        return buf[:n].view(shape)

    def check(self):
        for buf, n in self.bufs:
            if buf.dtype == torch.uint8:
                assert bool((buf[:n] != U8_FILL).all()), 'an output byte was not written'
                assert bool((buf[n:] == U8_FILL).all()), 'a kernel wrote past its output'
            else:
                assert not bool(torch.isnan(buf[:n]).any()), 'an output element was not written'
                assert bool(torch.isnan(buf[n:]).all()), 'a kernel wrote past its output'


# ------------------------------------------------------------------------------------------------- shared helpers
def _split(x):
    """fp32 -> round-to-nearest fp16 pair (hi, lo) with x ~= hi + lo."""
    hi = x.half()
    return hi, (x - hi.float()).half()


def _pair64(hi, lo):
    return hi.double() + lo.double()


def _split_emulated(v):
    """The kernels' st8_split of an fp32 value: hi = fp16(v), lo = fp16(v - hi)."""
    hi = v.half()
    return hi, (v - hi.float()).half()


def _ulp16(x):
    """Spacing of fp16 numbers at |x| (the subnormal step below 2^-14)."""
    a = x.abs().double().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def _report(name, err, bound):
    print(f'{name}: measured {err:.3e}, bound {bound:.3e}')
    assert err <= bound, (name, err, bound)


def _rel_err(got, ref):
    """max |got - ref| / max |ref|"""
    return float((got.double() - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


def _ulp_ratio(got, ref, slack):
    """max over elements of |got - ref| / (one fp16 ulp of ref + slack); <= 1 passes."""
    return float(((got.double() - ref).abs() / (_ulp16(ref) + slack)).max())


def _check_relu_hi(raw, raw_lo, relu):
    """Where the raw sum is positive the ReLU'd hi part equals raw's bit for bit; where it is negative it is 0."""
    s = raw.float() + raw_lo.float()
    pos, neg = s > 0, s < 0
    assert torch.equal(relu[pos], raw[pos])
    assert not bool(relu[neg].any())


# ------------------------------------------------------------------------------------------------- references
def _cbam_params(c, r, device, seed):
    g = torch.Generator(device=device).manual_seed(seed)
    return dict(w1=torch.randn(r, c, device=device, generator=g) / c**0.5,
                b1=torch.randn(r, device=device, generator=g) * 0.1,
                w2=torch.randn(c, r, device=device, generator=g) / r**0.5,
                b2=torch.randn(c, device=device, generator=g) * 0.1,
                ws=torch.randn(98, device=device, generator=g) * 0.1,
                bs=torch.randn(1, device=device, generator=g) * 0.1)


def _cbam_sd(p):
    """The kernels' CBAM parameters as the float64 state-dict entries oracle.network._cbam reads."""
    return {'a.ChannelGate.mlp.1.weight': p['w1'].double(), 'a.ChannelGate.mlp.1.bias': p['b1'].double(),
            'a.ChannelGate.mlp.3.weight': p['w2'].double(), 'a.ChannelGate.mlp.3.bias': p['b2'].double(),
            'a.SpatialGate.spatial.conv.weight': p['ws'].double().view(1, 2, 7, 7),
            'a.SpatialGate.spatial.conv.bias': p['bs'].double()}


def _cbam_residual_ref(sd, x64):
    """fp64 x + CBAM(x), NHWC in and out."""
    x = _nchw(x64)
    return _nhwc(x + onet._cbam(sd, 'a', x))


def _up2_ref(g64, skip64):
    """fp64 bilinear x2 (align_corners=False) of g [B,h,w,C] plus the broadcast skip [1,2h,2w,C]."""
    up = F.interpolate(_nchw(g64), scale_factor=2, mode='bilinear', align_corners=False)
    return _nhwc(up) + skip64


def _sum_parts_emulated(parts, res=None, res_lo=None):
    """sum_parts' fp32 arithmetic: parts 0 .. n-1 in order, then res, then res_lo, each a round-to-nearest add."""
    v = parts[0].clone()
    for p in range(1, parts.shape[0]):
        v = v + parts[p]
    if res is not None:
        v = v + res.float()
    if res_lo is not None:
        v = v + res_lo.float()
    return v


def _key_tail_emulated(y, ck):
    """key_tail's fixed-order fp32 sum of the partial sums y [parts, q, ld] -> (key, d, e)."""
    s = y[0].clone()
    for p in range(1, y.shape[0]):
        s = s + y[p]
    return s[:, :ck], s[:, ck], s[:, ck + 1:2 * ck + 1]


def _area_emulated(x, r):
    """area_down(_plane)'s fp32 arithmetic: the r x r window summed row by row from 0, times 1/r^2, then (for fp16 input)
    rounded to fp16.  x: [B,H,W,C] fp16 or [B,H,W] fp32."""
    plane = x.dim() == 3
    xx = x.unsqueeze(-1) if plane else x
    b, h, w, c = xx.shape
    v = xx.reshape(b, h // r, r, w // r, r, c)
    acc = torch.zeros(b, h // r, w // r, c, dtype=torch.float32, device=x.device)
    for dy in range(r):
        for dx in range(r):
            acc = acc + v[:, :, dy, :, dx, :].float()
    out = acc * (1.0 / (r * r))
    return out[..., 0] if plane else out.half()


def _area_ref(x64, r):
    """fp64 F.interpolate(mode='area') by 1/r of NHWC [B,H,W,C] or a plane [B,H,W]."""
    if x64.dim() == 3:
        return F.interpolate(x64.unsqueeze(1), scale_factor=1 / r, mode='area')[:, 0]
    return _nhwc(F.interpolate(_nchw(x64), scale_factor=1 / r, mode='area'))


def _head_taps(z):
    """The nine shifted tap planes of z [B,H,W,9] (zero padded): tap t = (dy+1)*3 + (dx+1) read at (y+dy, x+dx)."""
    b, h, w, _ = z.shape
    zp = F.pad(_nchw(z), (1, 1, 1, 1))
    return [zp[:, t, t // 3:t // 3 + h, t % 3:t % 3 + w] for t in range(9)]


def _head_emulated(z, bias):
    """head_gather3x3's fp32 arithmetic: bias, then taps 0..8 added in order (a padded tap adds 0)."""
    a = torch.full(z.shape[:3], bias, dtype=torch.float32, device=z.device)
    for tap in _head_taps(z):
        a = a + tap
    return a


def _head_ref(z, bias):
    """fp64 reference and the per-element magnitude sum |bias| + sum |z| of the taps."""
    taps = _head_taps(z.double())
    return bias + sum(taps), abs(bias) + sum(t.abs() for t in taps)


def _aggregate_emulated(logits):
    """aggregate_kernel's fp32 arithmetic: oracle.network.aggregate with the background product 1 - p_k taken in the
    kernel's fixed order k = 0 .. K-1."""
    p = torch.sigmoid(logits)
    bg = torch.ones_like(p[0])
    for k in range(p.shape[0]):
        bg = bg * (1 - p[k])
    full = torch.cat([bg.unsqueeze(0), p], 0).clamp(1e-7, 1 - 1e-7)
    return torch.log(full / (1 - full))


def _output_tail_ref(logits):
    """Reference of the output tail.  The aggregation stays in fp32, the network's arithmetic (oracle.network.aggregate
    casts to fp32; its 1 - p and its clamp to [1e-7, 1 - 1e-7] as fp32 constants are part of the operation), as both the
    oracle's form and the kernel's fixed-order emulation; bilinear x4 and softmax of the latter run in fp64.
    -> (agg emulated fp32 [K+1,h,w], agg oracle fp32, logits fp64 [K+1,4h,4w], prob fp64)."""
    agg = _aggregate_emulated(logits)
    up = F.interpolate(agg.double().unsqueeze(0), scale_factor=4, mode='bilinear', align_corners=False)[0]
    return agg, onet.aggregate(torch.sigmoid(logits), 0), up, torch.softmax(up, 0)


# ------------------------------------------------------------------------------------------------- CPU self-check
def test_reference_helpers_on_cpu():
    """The references and emulations above, on CPU at tiny shapes, against independent float64 formulations."""
    g = torch.Generator().manual_seed(0)
    # fp16 ulp
    ulp = _ulp16(torch.tensor([1.0, 0.75, 1e-6, 65504.0, -3.0]))
    assert ulp.tolist() == [2.0 ** -10, 2.0 ** -11, 2.0 ** -24, 32.0, 2.0 ** -9]
    # output placement: an unwritten element and a write into the guard are both caught
    outs = Outputs('cpu')
    y = outs.new((3, 4), torch.float32)
    y.fill_(1.0)
    outs.check()
    outs.bufs[0][0][12] = 0.0
    with pytest.raises(AssertionError):
        outs.check()
    outs = Outputs('cpu')
    outs.new((5,), torch.uint8)[:4] = 0
    with pytest.raises(AssertionError):
        outs.check()
    # hi/lo split
    x = torch.randn(1000, generator=g) * 10
    hi, lo = _split(x)
    # lo rounds to fp16: by 2^-11 of |lo| <= 2^-11 |x|, and to the subnormal step 2^-24 for small x
    assert bool(((_pair64(hi, lo) - x.double()).abs() <= 2.0 ** -22 * x.double().abs() + 2.0 ** -25).all())
    # sum_parts emulation against an fp64 sum
    parts = torch.randn(5, 4, 16, generator=g)
    res_hi, res_lo = _split(torch.randn(4, 16, generator=g))
    v = _sum_parts_emulated(parts, res_hi, res_lo)
    ref = parts.double().sum(0) + _pair64(res_hi, res_lo)
    assert float((v.double() - ref).abs().max()) < 8 * EPS32 * float(ref.abs().max())
    vh, vl = _split_emulated(v)
    assert float((_pair64(vh, vl) - ref).abs().max()) < 16 * EPS32 * float(ref.abs().max())
    assert torch.equal(_sum_parts_emulated(parts[:1]), parts[0])
    # key tail emulation
    y = torch.randn(3, 7, 2 * 4 + 1, generator=g)
    k, d, e = _key_tail_emulated(y, 4)
    s = y.double().sum(0)
    assert float((k.double() - s[:, :4]).abs().max()) < 1e-6 and float((d.double() - s[:, 4]).abs().max()) < 1e-6
    assert float((e.double() - s[:, 5:]).abs().max()) < 1e-6
    # area pooling: emulation and reference against a plain window mean
    xa = torch.randn(2, 8, 12, 16, generator=g).half()
    win = xa.double().view(2, 4, 2, 6, 2, 16).mean((2, 4))
    assert float((_area_ref(xa.double(), 2) - win).abs().max()) < 1e-12
    assert _ulp_ratio(_area_emulated(xa, 2), win, 0.0) < 0.501
    pl = torch.rand(2, 16, 8, generator=g)
    winp = pl.double().view(2, 4, 4, 2, 4).mean((2, 4))
    assert float((_area_ref(pl.double(), 4) - winp).abs().max()) < 1e-12
    assert float((_area_emulated(pl, 4).double() - winp).abs().max()) < 16 * 2.0 ** -24
    # the 3x3 gather as a convolution with one-hot taps
    z = torch.randn(2, 5, 6, 9, generator=g)
    onehot = torch.eye(9, dtype=torch.float64).view(1, 9, 3, 3)
    conv = F.conv2d(_nchw(z.double()), onehot, torch.tensor([0.25], dtype=torch.float64), padding=1)[:, 0]
    ref, mag = _head_ref(z, 0.25)
    assert float((ref - conv).abs().max()) < 1e-12
    assert float(((_head_emulated(z, 0.25).double() - conv).abs() / mag).max()) < 16 * EPS32
    # bilinear x2 reference at the border and inside: a constant field stays constant, a ramp stays linear inside
    ramp = torch.arange(6, dtype=torch.float64).view(1, 1, 6, 1).expand(1, 1, 6, 4).permute(0, 2, 3, 1)
    up = _up2_ref(ramp, torch.zeros(1, 12, 8, 1, dtype=torch.float64))
    assert torch.allclose(up[0, 1:11, 3, 0], torch.arange(1, 11, dtype=torch.float64) * 0.5 - 0.25)
    # output tail: probabilities sum to one; background log-odds from the product of the complements
    lg = torch.randn(3, 2, 3, generator=g) * 3
    agg, agg_oracle, lup, prob = _output_tail_ref(lg)
    assert float((prob.sum(0) - 1).abs().max()) < 1e-12
    assert float((agg - agg_oracle).abs().max()) < 1e-4
    bg = torch.prod(1 - torch.sigmoid(lg.double()), 0).clamp(1e-7, 1 - 1e-7)
    assert float((agg[0].double() - torch.log(bg / (1 - bg))).abs().max()) < 1e-4
    assert torch.equal(agg[1:], onet.aggregate(torch.sigmoid(lg), 0)[1:])


# ------------------------------------------------------------------------------------------------- CBAM
CBAM_CASES = [  # (C, B, h, w): 64 pixel slices; 256 / (C/8) pixel lanes per slice
    (512, 1, 4, 5), (512, 2, 7, 9), (512, 3, 13, 10), (512, 5, 30, 54), (512, 16, 68, 120),
    (64, 2, 30, 54), (2048, 2, 30, 54)]
CBAM_R = 32


def _cbam_inputs(c, b, h, w, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(b, h, w, c, device='cuda', generator=g) * 1.5 + torch.randn(c, device='cuda', generator=g) * 0.5
    return x, _cbam_params(c, CBAM_R, 'cuda', seed + 1)


def _cbam_scratch(b, h, w, c):
    from deva.model.native_ops import CBAM_POOL_SPLIT
    return torch.empty((2 * CBAM_POOL_SPLIT + 1) * b * c + 2 * b * h * w, dtype=torch.float32, device='cuda')


@pytest.mark.gpu
@pytest.mark.parametrize('c,b,h,w', CBAM_CASES)
def test_cbam_split(c, b, h, w):
    """x + CBAM(x) on the pair x = hi + lo, the gates pooled over x; raw as a pair, relu as hi."""
    nat = _nat()
    x, p = _cbam_inputs(c, b, h, w, 100 + c + b)
    hi, lo = _split(x)
    outs = Outputs()
    raw, raw_lo, relu = (outs.new((b, h, w, c), torch.float16) for _ in range(3))
    nat.cbam_split(hi, lo, p['w1'], p['b1'], p['w2'], p['b2'], p['ws'], p['bs'], _cbam_scratch(b, h, w, c), raw, raw_lo,
                   relu, b, h, w, c, CBAM_R)
    torch.cuda.synchronize()
    outs.check()
    ref = _cbam_residual_ref(_cbam_sd(p), _pair64(hi, lo))
    # fp32 pooling over up to 8160 pixels, the gate MLP and the 7x7 conv leave ~1e-7 relative; hi + lo holds the fp32
    # result to 2^-22 relative
    _report(f'cbam_split C={c} {b}x{h}x{w}: raw+lo rel', _rel_err(_pair64(raw, raw_lo), ref), 2e-6)
    _check_relu_hi(raw, raw_lo, relu)


# ------------------------------------------------------------------------------------------------- split-K finish
SUM_OUTPUTS = ['raw', 'raw+lo', 'relu', 'relu+lo', 'all']
SUM_SHAPE = (2, 30, 54, 64)


@pytest.mark.gpu
@pytest.mark.parametrize('outputs', SUM_OUTPUTS)
@pytest.mark.parametrize('residual', ['none', 'res', 'res+lo'])
@pytest.mark.parametrize('n_parts', [1, 2, 3, 4, 5])
def test_sum_parts(n_parts, residual, outputs):
    """Bit-exact against the fp32 emulation: parts 0..n-1 in order, then res, then res_lo; RN hi/lo conversions."""
    nat = _nat()
    shape = SUM_SHAPE
    g = torch.Generator(device='cuda').manual_seed(300 + n_parts)
    n = math.prod(shape)
    parts = torch.randn(n_parts, *shape, device='cuda', generator=g)
    res = res_lo = None
    if residual != 'none':
        res, lo = _split(torch.randn(*shape, device='cuda', generator=g) * 2)
        res_lo = lo if residual == 'res+lo' else None
    outs = Outputs()
    want_raw = outputs in ('raw', 'raw+lo', 'all')
    want_relu = outputs in ('relu', 'relu+lo', 'all')
    want_lo = outputs in ('raw+lo', 'relu+lo', 'all')
    raw = outs.new(shape, torch.float16) if want_raw else None
    raw_lo = outs.new(shape, torch.float16) if want_raw and want_lo else None
    relu = outs.new(shape, torch.float16) if want_relu else None
    relu_lo = outs.new(shape, torch.float16) if want_relu and want_lo else None
    nat.sum_parts(parts, n_parts, n, n, res=res, res_lo=res_lo, raw=raw, raw_lo=raw_lo, relu=relu, relu_lo=relu_lo)
    torch.cuda.synchronize()
    outs.check()
    v = _sum_parts_emulated(parts, res, res_lo)
    for got_hi, got_lo, val in ((raw, raw_lo, v), (relu, relu_lo, v.clamp_min(0))):
        if got_hi is None:
            continue
        hi, lo = _split_emulated(val)
        assert torch.equal(got_hi, hi)
        if got_lo is not None:
            assert torch.equal(got_lo, lo)


@pytest.mark.gpu
def test_sum_parts_grid_stride():
    """16 x 68 x 120 x 128 (1080p f8 at K = 16): more 8-channel vectors than threads, so the grid-stride loop runs more
    than once per thread."""
    nat = _nat()
    shape = (16, 68, 120, 128)
    n = math.prod(shape)
    threads = torch.cuda.get_device_properties(0).multi_processor_count * 32 * 256
    assert n // 8 > threads
    g = torch.Generator(device='cuda').manual_seed(310)
    parts = torch.randn(3, *shape, device='cuda', generator=g)
    res, res_lo = _split(torch.randn(*shape, device='cuda', generator=g))
    outs = Outputs()
    raw, raw_lo, relu, relu_lo = (outs.new(shape, torch.float16) for _ in range(4))
    nat.sum_parts(parts, 3, n, n, res=res, res_lo=res_lo, raw=raw, raw_lo=raw_lo, relu=relu, relu_lo=relu_lo)
    torch.cuda.synchronize()
    outs.check()
    v = _sum_parts_emulated(parts, res, res_lo)
    hi, lo = _split_emulated(v)
    assert torch.equal(raw, hi) and torch.equal(raw_lo, lo)
    hi, lo = _split_emulated(v.clamp_min(0))
    assert torch.equal(relu, hi) and torch.equal(relu_lo, lo)


# ------------------------------------------------------------------------------------------------- key projection tail
@pytest.mark.gpu
@pytest.mark.parametrize('n_parts', [1, 2, 7, 8])
@pytest.mark.parametrize('q', [20, 1620, 8160])
def test_key_tail(q, n_parts):
    """Partial sums [parts, q, 129] with part_stride = q * 129, as transform_key passes them: the key bit-exact against
    the fixed-order fp32 sum; shrinkage d^2 + 1 and selection sigmoid(e) within 1e-6 relative of fp64 applied to that
    sum (the kernel may contract d*d + 1 into an FMA, and it uses expf)."""
    nat = _nat()
    ck, ld = 64, 129
    g = torch.Generator(device='cuda').manual_seed(400 + q + n_parts)
    y = torch.randn(n_parts, q, ld, device='cuda', generator=g) * (2.0 / n_parts**0.5)
    outs = Outputs()
    key, sel = outs.new((q, ck), torch.float32), outs.new((q, ck), torch.float32)
    shr = outs.new((q,), torch.float32)
    nat.key_tail(y, ld, q, ck, key, shr, sel, n_parts=n_parts, part_stride=q * ld)
    torch.cuda.synchronize()
    outs.check()
    k, d, e = _key_tail_emulated(y, ck)
    assert torch.equal(key, k)
    d64 = d.double()
    shr_ref, sel_ref = d64 * d64 + 1, torch.sigmoid(e.double())
    _report(f'key_tail q={q} parts={n_parts}: shrinkage rel', float(((shr.double() - shr_ref).abs() / shr_ref).max()), 1e-6)
    _report(f'key_tail q={q} parts={n_parts}: selection rel', float(((sel.double() - sel_ref).abs() / sel_ref).max()), 1e-6)


# ------------------------------------------------------------------------------------------------- output tail
@pytest.mark.gpu
@pytest.mark.parametrize('k,h,w', [(1, 120, 216), (5, 120, 216), (31, 120, 216), (32, 120, 216), (33, 120, 216),
                                   (100, 120, 216), (33, 7, 13)])
def test_output_tail(k, h, w):
    """Aggregation, bilinear x4 and softmax.  K + 1 <= 32 keeps the logits in registers; K = 31 / 32 sit on either side
    of that path and K + 1 > 32 stashes them in prob.  About 10 % of the logits are +-30 (one in ten of them +30), so
    the clamps are exercised.  The others centre on -7, as in a frame where each object covers a small part: at K = 100
    the background then still holds most of the probability at some pixels, sits at its 1e-7 clamp at others, and lies
    in between elsewhere."""
    nat = _nat()
    g = torch.Generator(device='cuda').manual_seed(500 + k + h)
    logits = torch.randn(k, h, w, device='cuda', generator=g) * 2 - 7
    sat = torch.rand(k, h, w, device='cuda', generator=g) < 0.1
    sign = torch.where(torch.rand(k, h, w, device='cuda', generator=g) < 0.1, 30.0, -30.0)
    logits = torch.where(sat, sign, logits).contiguous()
    outs = Outputs()
    agg = outs.new((k + 1, h, w), torch.float32)
    prob = outs.new((k + 1, 4 * h, 4 * w), torch.float32)
    lgo = outs.new((k + 1, 4 * h, 4 * w), torch.float32)
    nat.output_tail(logits, agg, prob, lgo, k, h, w)
    torch.cuda.synchronize()
    outs.check()
    agg_ref, agg_oracle, lg_ref, prob_ref = _output_tail_ref(logits)
    assert float(prob_ref[0].max()) > 0.5 and float(prob_ref[1:].max()) > 0.5   # both kinds of pixel are present
    _report(f'output_tail K={k} {h}x{w}: aggregated log-odds abs', float((agg - agg_ref).abs().max()), 1e-5)
    # against the oracle's product order: K roundings of each product, amplified by 1 / (1 - bg) in log(bg / (1 - bg))
    c = agg_ref[0].sigmoid().double().clamp(1e-7, 1 - 1e-7)
    bound = 1e-5 + 2 * k * 2.0 ** -24 / (1 - c)
    _report(f'output_tail K={k} {h}x{w}: background log-odds vs aggregate / bound',
            float(((agg[0] - agg_oracle[0]).abs().double() / bound).max()), 1.0)
    assert float((agg[1:] - agg_oracle[1:]).abs().max()) <= 1e-5
    _report(f'output_tail K={k} {h}x{w}: logits abs', float((lgo.double() - lg_ref).abs().max()), 1e-4)
    _report(f'output_tail K={k} {h}x{w}: prob abs', float((prob.double() - prob_ref).abs().max()), 1e-5)
    _report(f'output_tail K={k} {h}x{w}: |sum prob - 1|', float((prob.double().sum(0) - 1).abs().max()), 1e-5)


# ------------------------------------------------------------------------------------------------- bilinear x2 + skip
UP2_CASES = ([(k, 30, 54, 512) for k in KS] + [(k, 60, 108, 256) for k in KS] +
             [(16, 68, 120, 512), (2, 1, 1, 8), (2, 2, 1, 64)])


def _up2_inputs(b, h, w, c, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(b, h, w, c, device='cuda', generator=g) * 3
    skip = torch.randn(1, 2 * h, 2 * w, c, device='cuda', generator=g)
    return x, skip


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['relu', 'relu_lo8'])
@pytest.mark.parametrize('b,h,w,c', UP2_CASES)
def test_up2_add_split_outputs(b, h, w, c, variant):
    """(g + g_lo) bilinear x2 + (skip + skip_lo): raw + raw_lo against fp64; the ReLU'd copy as fp16 against fp64, alone
    (relu: what up_16_8 consumes) or with its remainder as e4m3 of (x - fp16(x)) * 4096 (relu_lo8: up_8_4)."""
    nat = _nat()
    x, skip = _up2_inputs(b, h, w, c, 600 + b + h + c)
    hi, lo = _split(x)
    s_hi, s_lo = _split(skip)
    outs = Outputs()
    shape = (b, 2 * h, 2 * w, c)
    raw, raw_lo, relu = (outs.new(shape, torch.float16) for _ in range(3))
    relu_lo8 = outs.new(shape, torch.uint8) if variant == 'relu_lo8' else None
    nat.up2_add_split(hi, lo, s_hi, raw, raw_lo, relu, b, h, w, c, skip_lo=s_lo, relu_lo8=relu_lo8)
    torch.cuda.synchronize()
    outs.check()
    ref = _up2_ref(_pair64(hi, lo), _pair64(s_hi, s_lo))
    # fp32 interpolation of values ~10 (a few ulp) and the 2^-22 of the hi/lo pair
    _report(f'up2_add_split {shape} {variant}: raw+lo rel', _rel_err(_pair64(raw, raw_lo), ref), 2e-6)
    _check_relu_hi(raw, raw_lo, relu)
    # relu is one fp16 rounding of the fp32 value that raw + raw_lo holds to the bound above
    slack = 2e-6 * float(ref.abs().max())
    _report(f'up2_add_split {shape} {variant}: relu / (ulp16 + 2e-6 max|ref|)', _ulp_ratio(relu, ref.clamp_min(0), slack),
            1.0)
    if relu_lo8 is not None:  # 3-bit mantissa: <= 6.25 % + the e4m3 subnormal step, + the fp32 interpolation order
        rem = (ref.clamp_min(0) - relu.double()) * 4096.0
        got = relu_lo8.view(torch.float8_e4m3fn).double()
        bound = 0.07 * float(rem.abs().max()) + 2 ** -9 + 0.1
        _report(f'up2_add_split {shape}: e4m3 remainder abs', float((got - rem).abs().max()), bound)


# ------------------------------------------------------------------------------------------------- max pool
@pytest.mark.gpu
@pytest.mark.parametrize('b,h,w,c,pair', [(1, 240, 432, 64, True), (5, 240, 432, 64, False), (2, 33, 47, 64, True),
                                          (2, 33, 47, 64, False)])
def test_maxpool(b, h, w, c, pair):
    """3x3 / 2 / pad 1 max pool, bit-exact: y = fp16(max(hi + lo)), y_lo = fp16(m - y) (pair) or y = max(x) (single)."""
    nat = _nat()
    g = torch.Generator(device='cuda').manual_seed(800 + b + h)
    x = torch.randn(b, h, w, c, device='cuda', generator=g) * 4
    hi, lo = _split(x)
    ho, wo = (h + 1) // 2, (w + 1) // 2
    outs = Outputs()
    y = outs.new((b, ho, wo, c), torch.float16)
    y_lo = outs.new((b, ho, wo, c), torch.float16) if pair else None
    nat.maxpool(hi, y, b, h, w, c, x_lo=lo if pair else None, y_lo=y_lo)
    torch.cuda.synchronize()
    outs.check()
    src = hi.float() + lo.float() if pair else hi.float()
    m = _nhwc(F.max_pool2d(_nchw(src), 3, 2, 1))
    want_hi, want_lo = _split_emulated(m)
    assert torch.equal(y, want_hi)
    if pair:
        assert torch.equal(y_lo, want_lo)


# ------------------------------------------------------------------------------------------------- area down-sampling
@pytest.mark.gpu
@pytest.mark.parametrize('k', KS)
@pytest.mark.parametrize('r,h,w', [(2, 60, 108), (4, 120, 216)])
def test_area_down(r, h, w, k):
    """r x r mean of fp16 [K,h,w,256]: bit-exact against the fp32 emulation and within one fp16 ulp of fp64."""
    nat = _nat()
    c = 256
    g = torch.Generator(device='cuda').manual_seed(900 + r + k)
    x = (torch.randn(k, h, w, c, device='cuda', generator=g) * 2).half()
    outs = Outputs()
    y = outs.new((k, h // r, w // r, c), torch.float16)
    nat.area_down(x, y, k, h, w, c, r)
    torch.cuda.synchronize()
    outs.check()
    assert torch.equal(y, _area_emulated(x, r))
    _report(f'area_down r={r} K={k}: err / ulp16', _ulp_ratio(y, _area_ref(x.double(), r), 0.0), 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize('k', KS)
@pytest.mark.parametrize('r,h,w', [(16, 480, 864), (4, 120, 216)])
def test_area_down_plane(r, h, w, k):
    """r x r mean of fp32 planes [K,h,w] (masks at r = 16, logits at r = 4): bit-exact against the fp32 emulation, and
    within (r^2 - 1) * 2^-24 of the window's mean |x| from fp64 - the bound of a sequential fp32 sum of r^2 terms (an
    add rounds by at most 2^-24 of the partial sum); the multiply by 1 / r^2 is exact."""
    nat = _nat()
    g = torch.Generator(device='cuda').manual_seed(950 + r + k)
    x = torch.rand(k, h, w, device='cuda', generator=g) if r == 16 else torch.randn(k, h, w, device='cuda', generator=g) * 5
    outs = Outputs()
    y = outs.new((k, h // r, w // r), torch.float32)
    nat.area_down_plane(x, y, k, h, w, r)
    torch.cuda.synchronize()
    outs.check()
    assert torch.equal(y, _area_emulated(x, r))
    ref = _area_ref(x.double(), r)
    mag = _area_ref(x.double().abs(), r)
    _report(f'area_down_plane r={r} K={k}: err / mean|x|', float(((y.double() - ref).abs() / mag).max()),
            (r * r - 1) * 2.0 ** -24)


# ------------------------------------------------------------------------------------------------- fused head gather
@pytest.mark.gpu
@pytest.mark.parametrize('b,h,w', [(1, 120, 216), (5, 120, 216), (16, 120, 216), (3, 1, 1), (2, 2, 3)])
def test_head_gather3x3(b, h, w):
    """bias + the nine zero-padded taps of z [B,H,W,9]: bit-exact against the fp32 order, within 1e-6 x sum |z| of fp64."""
    nat = _nat()
    g = torch.Generator(device='cuda').manual_seed(1000 + b + h)
    z = torch.randn(b, h, w, 9, device='cuda', generator=g) * 3
    bias = -0.37
    outs = Outputs()
    out = outs.new((b, h, w), torch.float32)
    nat.head_gather3x3(z, out, bias, b, h, w)
    torch.cuda.synchronize()
    outs.check()
    assert torch.equal(out, _head_emulated(z, bias))
    ref, mag = _head_ref(z, bias)
    _report(f'head_gather3x3 {b}x{h}x{w}: err / sum|z|', float(((out.double() - ref).abs() / mag).max()), 1e-6)


# ------------------------------------------------------------------------------------------------- value append
@pytest.mark.gpu
@pytest.mark.parametrize('n', [1620, 8160])
def test_transpose_append(n):
    """Token-major [n, 512] fp16 -> bank columns 37 .. 37 + n - 1 of rows with ld = cap > n: exact, and the columns on
    both sides (and the memory after the bank) untouched."""
    nat = _nat()
    c, col0 = 512, 37
    cap = col0 + n + 27
    g = torch.Generator(device='cuda').manual_seed(1100 + n)
    src = torch.randn(n, c, device='cuda', generator=g).half()
    buf = torch.randn(c * cap + GUARD, device='cuda', generator=g).half()
    before = buf.clone()
    nat.transpose_append(src, buf[col0:], cap, n, c)
    torch.cuda.synchronize()
    bank, old = buf[:c * cap].view(c, cap), before[:c * cap].view(c, cap)
    assert torch.equal(bank[:, col0:col0 + n], src.t())
    assert torch.equal(bank[:, :col0], old[:, :col0]) and torch.equal(bank[:, col0 + n:], old[:, col0 + n:])
    assert torch.equal(buf[c * cap:], before[c * cap:])
