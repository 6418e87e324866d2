"""The staged convolution epilogue (residual read from the TMA ring, outputs drained by TMA stores) writes exactly what
the per-thread epilogue writes, bit for bit, and nothing outside the output tensors.

Every case runs the same launch twice: once with DEVA_B200_CONV_EPI=staged (the library refuses the launch rather than
fall back, so the staged epilogue is known to have run) and once with DEVA_B200_CONV_EPI=regs.  Outputs are NaN-filled
buffers followed by a guard region, so an element the staged stores miss or a store past the end shows.  The 4x4 pool
of the raw output that the staged epilogue can emit (`out_pool4`) equals area_down(raw, 4) bit for bit.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GUARD = 4096  # elements after each output

CASES = [
    # id, b, h, w, cin, cout, k, residual ('own' / 'broadcast' / None), outputs, head, rank-1
    ('n64_full', 2, 32, 64, 64, 64, 3, 'own', ('raw', 'relu'), False, False),
    ('n128_full', 2, 32, 64, 128, 128, 3, None, ('relu',), False, False),
    ('n192_full', 2, 32, 64, 64, 192, 3, 'own', ('raw',), False, False),
    ('n256_full', 2, 32, 64, 64, 256, 3, 'own', ('raw', 'raw_lo'), False, False),
    ('edges_hw', 3, 37, 45, 64, 256, 3, 'own', ('raw', 'relu', 'relu_lo'), False, False),
    ('broadcast', 4, 29, 61, 128, 256, 3, 'broadcast', ('raw',), False, False),
    ('two_tiles_1x1', 2, 34, 50, 128, 512, 1, 'own', ('relu', 'relu_lo8'), False, False),
    ('many_tiles', 3, 100, 150, 64, 128, 3, 'own', ('relu',), False, False),
    ('relu_lo8', 2, 40, 72, 128, 256, 3, None, ('relu', 'relu_lo8'), False, False),
    ('res_relu_lo8', 2, 27, 33, 128, 128, 1, 'own', ('relu', 'relu_lo8'), False, False),
    ('res_hi_only', 3, 37, 45, 64, 256, 3, 'own_hi', ('raw', 'relu'), False, False),
    ('res_hi_only_lo8', 2, 27, 33, 128, 128, 1, 'own_hi', ('relu', 'relu_lo8'), False, False),
    ('res_hi_only_lo8_alone', 2, 27, 33, 128, 128, 1, 'own_hi', ('relu_lo8',), False, False),
    ('head_only', 2, 37, 45, 64, 256, 3, 'own', (), True, False),
    ('rank1', 2, 31, 47, 65, 128, 1, None, ('raw', 'relu'), False, True),
]


def _run(x, pc, kw, outs, head_w, rank1_x, regs, pool4=None, tile=None):
    from deva import _native as nat
    from deva.model import native_ops as ops
    b, h, w, _ = x.shape
    ho, wo = pc.out_hw(h, w)
    th, tw = tile or ops.choose_tile(ho, wo)
    n = b * ho * wo * pc.cout
    bufs = {}
    for name in outs:
        if name == 'relu_lo8':
            bufs[name] = torch.full((n + GUARD,), 0xFF, dtype=torch.uint8, device='cuda')  # 0xFF: e4m3 NaN
        else:
            bufs[name] = torch.full((n + GUARD,), float('nan'), dtype=torch.float16, device='cuda')
    head_out = None
    if head_w is not None:
        head_out = torch.full((b * ho * wo * head_w.shape[0] + GUARD,), float('nan'), device='cuda')
    old = os.environ.get('DEVA_B200_CONV_EPI')
    os.environ['DEVA_B200_CONV_EPI'] = 'regs' if regs else 'staged'
    try:
        nat.conv2d(x, b, h, w, pc.cin_pad, pc.w_packed, pc.k, pc.stride, pc.cout, pc.cout_pad, pc.nt, th, tw, pc.bias,
                   rank1_w=pc.rank1_w, rank1_x=rank1_x, out_raw=bufs.get('raw'), out_relu=bufs.get('relu'),
                   out_raw_lo=bufs.get('raw_lo'), out_relu_lo=bufs.get('relu_lo'), out_relu_lo8=bufs.get('relu_lo8'),
                   head_w=head_w, head_out=head_out, head_n=0 if head_w is None else head_w.shape[0],
                   x_lo8=kw.get('x_lo8'), w8_packed=pc.w8_packed, acc_scale=pc.acc_scale, split_mode=pc.split_mode,
                   res=kw.get('res'), res_lo=kw.get('res_lo'), res_broadcast=kw.get('res_broadcast', False),
                   out_pool4=pool4)
    finally:
        if old is None:
            os.environ.pop('DEVA_B200_CONV_EPI', None)
        else:
            os.environ['DEVA_B200_CONV_EPI'] = old
    torch.cuda.synchronize()
    if head_out is not None:
        bufs['head'] = head_out
    return bufs, n


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else (t.view(torch.int32) if t.dtype == torch.float32 else t)


def _check_same(staged, regs, n, head_len=None):
    for name, s in staged.items():
        r = regs[name]
        end = head_len if name == 'head' else n
        body, guard = s[:end], s[end:]
        if name == 'relu_lo8':
            assert not bool((body == 0xFF).any()), f'{name}: element not written'
            assert bool((guard == 0xFF).all()), f'{name}: written past the end'
        else:
            assert not bool(torch.isnan(body).any()), f'{name}: element not written'
            assert bool(torch.isnan(guard).all()), f'{name}: written past the end'
        assert torch.equal(_bits(body), _bits(r[:end])), f'{name}: staged and per-thread epilogues differ'


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_staged_epilogue_matches_register_epilogue(case):
    from deva import _native as nat
    from deva.model import native_ops as ops
    nat.require_device()
    _, b, h, w, cin, cout, k, res_kind, outs, head, rank1 = case
    g = torch.Generator(device='cuda').manual_seed(b * 7919 + h * 31 + cout + k)
    wgt = torch.randn(cout, cin, k, k, device='cuda', generator=g) / (cin * k * k)**0.5
    bias = torch.randn(cout, device='cuda', generator=g)
    pc = ops.PackedConv(wgt, bias, 1, rank1_in=0 if rank1 else None)
    x = torch.randn(b, h, w, pc.cin_pad, device='cuda', generator=g).half()
    kw = {}
    if res_kind is not None:
        r = torch.randn(1 if res_kind == 'broadcast' else b, h, w, cout, device='cuda', generator=g)
        kw['res'] = r.half()
        if res_kind != 'own_hi':
            kw['res_lo'] = (r - kw['res'].float()).half()
        kw['res_broadcast'] = res_kind == 'broadcast'
    head_w = torch.randn(9, cout, device='cuda', generator=g) / cout**0.5 if head else None
    rank1_x = torch.randn(b, h * w, device='cuda', generator=g) if rank1 else None
    staged, n = _run(x, pc, kw, outs, head_w, rank1_x, regs=False)
    regs, _ = _run(x, pc, kw, outs, head_w, rank1_x, regs=True)
    _check_same(staged, regs, n, None if head_w is None else b * h * w * 9)


def test_staged_epilogue_matches_in_the_parity_form_of_up_8_4_c2():
    """e4m3 correction pass, (hi, lo) residual, raw output and the fused head, on 4x32 tiles with edges."""
    from deva import _native as nat
    from deva.model import native_ops as ops
    nat.require_device()
    b, h, w, c = 3, 30, 70, 256
    g = torch.Generator(device='cuda').manual_seed(84)
    wgt = torch.randn(c, c, 3, 3, device='cuda', generator=g) / (c * 9)**0.5
    pc = ops.PackedConv(wgt, torch.randn(c, device='cuda', generator=g), 1, act_lo8=True)
    x = torch.randn(b, h, w, c, device='cuda', generator=g).half()
    r = torch.randn(b, h, w, c, device='cuda', generator=g)
    kw = dict(x_lo8=(torch.randn(b, h, w, c, device='cuda', generator=g) * 4).to(torch.float8_e4m3fn).view(torch.uint8),
              res=r.half(), res_lo=(r - r.half().float()).half())
    head_w = torch.randn(9, c, device='cuda', generator=g) / c**0.5
    for outs in (('raw',), ()):
        staged, n = _run(x, pc, kw, outs, head_w, None, regs=False)
        regs, _ = _run(x, pc, kw, outs, head_w, None, regs=True)
        _check_same(staged, regs, n, b * h * w * 9)


def _pool_case(b, h, w, seed, act_lo8=False):
    from deva.model import native_ops as ops
    c = 256
    g = torch.Generator(device='cuda').manual_seed(seed)
    wgt = torch.randn(c, c, 3, 3, device='cuda', generator=g) / (c * 9)**0.5
    pc = ops.PackedConv(wgt, torch.randn(c, device='cuda', generator=g), 1, act_lo8=act_lo8)
    x = torch.randn(b, h, w, c, device='cuda', generator=g).half()
    r = torch.randn(b, h, w, c, device='cuda', generator=g)
    kw = dict(res=r.half(), res_lo=(r - r.half().float()).half())
    if act_lo8:
        kw['x_lo8'] = (torch.randn(b, h, w, c, device='cuda', generator=g) * 4).to(torch.float8_e4m3fn).view(torch.uint8)
    head_w = torch.randn(9, c, device='cuda', generator=g) / c**0.5
    return pc, x, kw, head_w


@pytest.mark.parametrize('b,h,w,act_lo8', [(3, 32, 96, True), (2, 44, 100, False), (4, 8, 32, True)])
def test_pool4_equals_area_down_of_the_raw_output(b, h, w, act_lo8):
    """c2's form: the pool with and without the raw output, against area_down of the raw output, several tiles."""
    from deva import _native as nat
    from deva.model import native_ops as ops
    nat.require_device()
    pc, x, kw, head_w = _pool_case(b, h, w, b * 100 + h, act_lo8)
    tile = ops.choose_tile(h, w, pool4=True)
    n_pool = b * (h // 4) * (w // 4) * pc.cout
    pool = torch.full((n_pool + GUARD,), float('nan'), dtype=torch.float16, device='cuda')
    both, n = _run(x, pc, kw, ('raw',), head_w, None, regs=False, pool4=pool, tile=tile)
    want = ops.area_down(both['raw'][:n].view(b, h, w, pc.cout), 4).reshape(-1)
    assert bool(torch.isnan(pool[n_pool:]).all()), 'pool written past the end'
    assert torch.equal(pool[:n_pool].view(torch.int16), want.view(torch.int16))
    pool_only = torch.full_like(pool, float('nan'))
    alone, _ = _run(x, pc, kw, (), head_w, None, regs=False, pool4=pool_only, tile=tile)
    assert torch.equal(pool_only.view(torch.int16), pool.view(torch.int16))
    assert torch.equal(alone['head'].view(torch.int32), both['head'].view(torch.int32))
    regs, _ = _run(x, pc, kw, ('raw',), head_w, None, regs=True, tile=tile)
    assert torch.equal(regs['raw'].view(torch.int16), both['raw'].view(torch.int16))
    assert torch.equal(regs['head'].view(torch.int32), both['head'].view(torch.int32))


@pytest.mark.parametrize('h,w,tile', [(30, 64, (4, 32)), (32, 66, (4, 32)), (32, 64, (2, 64))])
def test_pool4_is_refused_off_the_4_grid(h, w, tile):
    from deva import _native as nat
    nat.require_device()
    pc, x, kw, head_w = _pool_case(2, h, w, 7)
    pool = torch.empty(2 * (h // 4) * (w // 4) * pc.cout, dtype=torch.float16, device='cuda')
    with pytest.raises(RuntimeError, match='out_pool4'):
        _run(x, pc, kw, ('raw',), head_w, None, regs=False, pool4=pool, tile=tile)
