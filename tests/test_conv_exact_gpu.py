"""The convolution kernel against oracle/conv_desc.py with zero tolerance, on exactly representable operands.

Every operand sits on a small dyadic grid: activations are small integers, weights are in {-1, 0, 1}, and the low-order
operands (x_lo, the weights' lo half), the bias, the rank-1 term and res_lo are multiples of 2^-g (coarser for the
low-order passes); the e4m3 operands are small integers and acc_scale a power of two.  Each case asserts, as a
precondition, that M * 2^g <= 2^22 for every element (M: the oracle's magnitude, the sum of |term|), so every partial
sum in any order is an fp32 number with margin, and for the fp8 pass that its e4m3 sum stays below 2^13 (wgmma adds e4m3
products with a ~14-bit adder).  The kernel's fp32 result must then equal the float64 value bit for bit, whatever order
the tensor cores add in, and every fp16 / e4m3 output must be the exact conversion of it.  A wrong tap, channel block,
weight column, bias or residual channel, chain bound, pass or scale moves some element by at least 2^-g.

That wgmma's fp32 accumulation is exact on such sums is measured, not assumed: on an H100 80GB HBM3 every case of every
mode, fp16 and e4m3 passes alike, matched the float64 value bit for bit, so no case falls back to a looser bound.  A
mismatch is reported with its (image, y, x, channel, chain) and its size next to one fp32 ulp of M.

The operands are built directly (hi, lo and e4m3 parts with nonzero low-order passes) rather than through PackedConv.
Each case runs through nat.conv2d with its tile and channel tile forced, once with DEVA_B200_CONV_EPI=staged where the
launch takes the staged epilogue and once with =regs (per-thread); outputs are NaN-filled (0xFF for bytes) buffers
followed by a guard region.  The gate outputs go through the fast sigmoid / tanh, so they are compared with the float64
update of the exact pre-activations to one fp16 ulp + 2e-6.  The cases are tests/golden/conv_cases.py.
"""
import os
import sys
import time

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
from conv_cases import CASES, SPLIT_PARTS  # noqa: E402

from oracle import conv_desc as cd  # noqa: E402

pytestmark = pytest.mark.gpu

GUARD = 4096
NT_MMA = (64, 128, 192, 256)


def _takes_staged(c):
    """The staged epilogue's conditions (conv.cu plan_staged) for the case's launch."""
    if c.get('gates') or c.get('ksplit', 0) > 1 or 'f32' in c['outs'] or c['nt'] not in NT_MMA:
        return False
    cout_pad = -(-c['cout'] // c['nt']) * c['nt']
    if c['cout'] != cout_pad:
        return False
    n16 = sum(o in c['outs'] for o in ('raw_lo', 'relu', 'relu_lo')) + int('raw' in c['outs'] or bool(c.get('pool4')))
    if 'relu_lo8' in c['outs']:
        return max(n16, 1 if c.get('res') else 0, 2 if c.get('res_lo') else 0) <= 2
    return n16 <= 3


PARAMS = [(name, epi) for name, c in CASES.items() for epi in ('staged', 'regs')
          if epi == 'regs' and not c.get('pool4') or epi == 'staged' and _takes_staged(c)]


def _grid(shape, lo, hi, step, g, dtype, p_nonzero=1.0):
    """Uniform integers in [lo, hi] times `step`, as `dtype` (exact), on the device."""
    v = torch.randint(lo, hi + 1, shape, generator=g, device='cuda').double() * step
    if p_nonzero < 1:
        v = v * (torch.rand(shape, generator=g, device='cuda') < p_nonzero)
    out = v.to(dtype)
    assert torch.equal(out.double(), v), 'grid value not representable'
    return out


def _e4m3(shape, lo, hi, g):
    v = torch.randint(lo, hi + 1, shape, generator=g, device='cuda').float()
    return v.to(torch.float8_e4m3fn).view(torch.uint8)


def _operands(name):
    """The launch's keyword arguments (outputs NaN-filled with a guard region) and the case."""
    c = CASES[name]
    g = torch.Generator(device='cuda').manual_seed(sum(map(ord, name)))
    b, h, w, cin_pad, cout, k, s, nt = (c[x] for x in ('b', 'h', 'w', 'cin_pad', 'cout', 'k', 's', 'nt'))
    gexp = c.get('g', 10)
    hexp = gexp // 2
    cout_pad = -(-cout // nt) * nt
    taps = k * k
    ho, wo = (h + 2 * (k // 2) - k) // s + 1, (w + 2 * (k // 2) - k) // s + 1
    mode = c['mode']
    sparse = c.get('sparse', False)
    xr = 1 if sparse else 2
    pw = 1 / 64 if sparse else 1.0
    f16 = torch.float16
    act = lambda: _grid((b, h, w, cin_pad), -xr, xr, 1.0, g, f16)  # noqa: E731
    groups = 2 if mode in ('x2', 'x_lo', 'w_lo') else 1
    wp = torch.empty(cout_pad, groups, taps, cin_pad, dtype=f16, device='cuda')
    wp[:, 0] = _grid((cout_pad, taps, cin_pad), -1, 1, 1.0, g, f16, pw)
    if groups == 2:
        wp[:, 1] = (_grid((cout_pad, taps, cin_pad), -1, 1, 1.0, g, f16, pw) if mode == 'x2'
                    else _grid((cout_pad, taps, cin_pad), -8, 8, 2.0 ** -hexp, g, f16))
    kw = dict(x=act(), batch=b, h=h, w=w, cin_pad=cin_pad, w_packed=wp.view(cout_pad, -1), kh=k, stride=s, cout=cout,
              cout_pad=cout_pad, nt=nt, th=0 if c['tile'] == 'flat' else c['tile'][0],
              tw=128 if c['tile'] == 'flat' else c['tile'][1],
              bias=_grid((cout_pad,), -2 ** (gexp + 1), 2 ** (gexp + 1), 2.0 ** -gexp, g, torch.float32))
    if mode == 'x2':
        kw['x2'] = act()
    elif mode == 'x_lo':
        kw['x_lo'] = _grid((b, h, w, cin_pad), -8, 8, 2.0 ** -hexp, g, f16)
    elif mode == 'w_lo':
        kw['split_mode'] = 2
    elif mode == 'lo8':
        kw.update(split_mode=3, x_lo8=_e4m3((b, h, w, cin_pad), -3, 3, g),
                  w8_packed=_e4m3((cout_pad, taps * cin_pad), -2, 2, g), acc_scale=0.25)
    if c.get('rank1'):
        kw['rank1_w'] = _grid((cout_pad,), -4, 4, 0.25, g, torch.float32)
        kw['rank1_x'] = _grid((b * ho * wo,), -2 ** (gexp - 1), 2 ** (gexp - 1), 2.0 ** (2 - gexp), g, torch.float32)
    if c.get('res'):
        rb = 1 if c['res'] == 'broadcast' else b
        kw['res'] = _grid((rb, ho, wo, cout), -4, 4, 1.0, g, f16)
        kw['res_broadcast'] = rb == 1 and b > 1
        if c.get('res_lo'):
            kw['res_lo'] = _grid((rb, ho, wo, cout), -2 ** max(gexp - 4, 0), 2 ** max(gexp - 4, 0), 2.0 ** -gexp, g, f16)
    if c.get('ksplit'):
        kw['ksplit'] = c['ksplit']
    n = b * ho * wo * cout
    parts = len(cd.k_layout(kw)[2])
    for o in c['outs']:
        if o == 'relu_lo8':
            kw['out_relu_lo8'] = torch.full((n + GUARD,), 0xFF, dtype=torch.uint8, device='cuda')
        elif o == 'f32':
            kw['out_f32'] = torch.full((parts * n + GUARD,), float('nan'), device='cuda')
        else:
            kw['out_' + o] = torch.full((n + GUARD,), float('nan'), dtype=f16, device='cuda')
    if c.get('head_n'):
        kw['head_n'] = c['head_n']
        kw['head_w'] = _grid((c['head_n'], cout), -1, 1, 1.0, g, torch.float32)
        kw['head_out'] = torch.full((b * ho * wo * c['head_n'] + GUARD,), float('nan'), device='cuda')
    if c.get('gates'):
        kw['gate_h'] = torch.randn(b, ho, wo, cout // 3, generator=g, device='cuda').half()
        kw['gate_out'] = torch.full((n // 3 + GUARD,), float('nan'), dtype=f16, device='cuda')
    if c.get('pool4'):
        kw['out_pool4'] = torch.full((n // 16 + GUARD,), float('nan'), dtype=f16, device='cuda')
    return kw, c, gexp


def _run(kw, epi):
    old = os.environ.get('DEVA_B200_CONV_EPI')
    os.environ['DEVA_B200_CONV_EPI'] = epi
    try:
        from deva import _native as nat
        nat.conv2d(**kw)
        torch.cuda.synchronize()
    finally:
        if old is None:
            os.environ.pop('DEVA_B200_CONV_EPI')
        else:
            os.environ['DEVA_B200_CONV_EPI'] = old


def _where(o, flat, cout, per_pixel=None):
    """(image, y, x, channel, chain) of flat element `flat` of a [chains, pixels, cout] comparison."""
    per_pixel = per_pixel or cout
    pixels = o.pix.numel()
    chain, rest = divmod(flat, pixels * per_pixel)
    p, ch = divmod(rest, per_pixel)
    q = int(o.pix[p])
    return dict(image=q // (o.ho * o.wo), y=q // o.wo % o.ho, x=q % o.wo, channel=ch, chain=chain)


_BITS = {torch.float16: torch.int16, torch.float32: torch.int32, torch.uint8: torch.uint8}


def _check_bits(name, what, got, want, o, cout):
    g, w_ = got.reshape(-1).view(_BITS[got.dtype]), want.reshape(-1).view(_BITS[want.dtype])
    bad = (g != w_).nonzero()
    if bad.numel():
        i = int(bad[0])
        per_pixel = want.shape[-1]
        loc = _where(o, i, cout, per_pixel)
        gv, wv = got.reshape(-1)[i].item(), want.reshape(-1)[i].item()
        ulp = ''
        if what in ('f32', 'raw'):
            m = float(o.chain_mag.reshape(-1)[i]) if what == 'f32' else float(o.mag.reshape(-1)[i])
            ulp = f'; |diff| {abs(gv - wv):.3e} vs one fp32 ulp of M {torch.finfo(torch.float32).eps * m:.3e}'
        raise AssertionError(f'{name}: {what} differs in {bad.numel()} of {g.numel()} elements; first at {loc}: '
                             f'kernel {gv!r}, oracle {wv!r}{ulp}')


@pytest.fixture(scope='module', autouse=True)
def _duration():
    from deva import _native
    _native.require_device()
    t0 = time.perf_counter()
    yield
    print(f'\ntest_conv_exact_gpu.py: {len(PARAMS)} launches, {time.perf_counter() - t0:.1f} s')


@pytest.mark.parametrize('name,epi', PARAMS)
def test_exact(name, epi):
    kw, c, gexp = _operands(name)
    o = cd.launch(**kw)
    # precondition: every partial sum of every element is an exact fp32 number with margin
    lim = 2.0 ** (22 - gexp)
    assert float(o.chain_mag.max()) <= lim, f'{name}: M {float(o.chain_mag.max())} > 2^{22 - gexp}'
    if o.mag8 is not None:
        assert float(o.mag8.max()) <= 2 ** 13, f'{name}: e4m3 sum {float(o.mag8.max())}'
    if 'head_mag' in o.outputs:
        assert float(o.outputs['head_mag'].max()) <= lim
    if name in SPLIT_PARTS:
        assert len(o.chains) == SPLIT_PARTS[name]
    assert torch.equal(o.value.float().double(), o.value), 'value not exact in fp32'
    _run(kw, epi)
    cout = c['cout']
    n_el = o.pix.numel() * cout
    for what, want in o.outputs.items():
        if what in ('head_mag', 'gate_h', 'pool4_win'):
            continue
        key = {'head': 'head_out', 'gate': 'gate_out', 'pool4': 'out_pool4'}.get(what, 'out_' + what)
        buf = kw[key]
        body, guard = buf[:-GUARD], buf[-GUARD:]
        if buf.dtype == torch.uint8:
            assert bool((guard == 0xFF).all()), f'{name}: {what} guard region written'
        else:
            assert bool(guard.isnan().all()), f'{name}: {what} guard region written'
        if what == 'gate':
            got = body.view(-1, cout // 3).double()
            tol = (want.abs() * 2.0 ** -10).clamp_min(2.0 ** -24) + 2e-6  # one fp16 ulp (>= its spacing) + 2e-6
            err = (got - want).abs()
            assert not got.isnan().any(), f'{name}: gate output not written'
            if bool((err > tol).any()):
                i = int((err - tol).reshape(-1).argmax())
                raise AssertionError(f'{name}: gate off by {float(err.reshape(-1)[i]):.3e} at '
                                     f'{_where(o, i, cout // 3)} (f, u, n pre-activations exact)')
            continue
        if what == 'head':
            assert torch.equal(o.value.float().double().clamp_min(0) @ kw['head_w'].double().t(), want)
            want = want.float()
        _check_bits(name, what, body.view(want.shape), want, o, cout)
    if 'f32' in o.outputs:
        assert o.outputs['f32'].numel() == len(o.chains) * n_el


def test_gate_epilogue_refuses_a_scaled_accumulator():
    """The gate epilogue evaluates the gates on the unscaled accumulator: a launch that asks for acc_scale != 1 with it
    is refused rather than computed unscaled."""
    kw, _, _ = _operands('gates_flat')
    kw['acc_scale'] = 0.5
    with pytest.raises(RuntimeError, match='gate'):
        _run(kw, 'regs')
