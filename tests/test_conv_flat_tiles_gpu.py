"""Flat pixel tiles (128 consecutive output pixels of one image, im2col-mode activation loads) and narrower channel tiles
write exactly what the rectangular tiles and the packed channel tile write, bit for bit, and nothing else.

Every case launches the same convolution through nat.conv2d with flat tiles (th = 0, tw = 128) and with the best
rectangle, in the epilogue form the launch takes by itself and in the per-thread form (DEVA_B200_CONV_EPI=regs).  The
outputs are NaN-filled buffers followed by a guard region, so a row past an image's last pixel that reached memory, or
an element no store wrote, shows up in the comparison.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GUARD = 4096  # elements after each output

# id: (batch, h, w, cin, cout, k, mode)
CASES = {
    '1x1_b16': (16, 68, 120, 256, 256, 1, 'raw'),
    '3x3_b16_relu': (16, 68, 120, 128, 256, 3, 'relu'),
    '3x3_b1_relu': (1, 68, 120, 256, 256, 3, 'relu'),
    '3x3_c2_res': (4, 30, 54, 128, 256, 3, 'res'),
    'ragged_res_broadcast': (4, 37, 53, 128, 256, 3, 'res_broadcast'),
    'ragged_two_inputs': (2, 37, 53, 256, 256, 3, 'two'),
    'gates_b16': (16, 68, 120, 256, 384, 3, 'gates'),
    'precise_splitk_b1': (1, 68, 120, 256, 256, 3, 'precise_splitk'),
    'precise_1x1': (2, 30, 54, 128, 256, 1, 'precise'),
    'act_lo8_b1': (1, 68, 120, 256, 256, 3, 'lo8'),
    'act_lo8_res': (2, 37, 53, 128, 256, 3, 'lo8_res'),
    'rank1': (2, 37, 53, 65, 128, 1, 'rank1'),
    'head': (2, 68, 120, 64, 256, 3, 'head'),
    'odd_cout_f32': (2, 37, 53, 64, 33, 3, 'f32'),
}


def _inputs(name, nt_override=None):
    from deva.model import native_ops as ops
    b, h, w, cin, cout, k, mode = CASES[name]
    g = torch.Generator(device='cuda').manual_seed(sum(map(ord, name)))
    two = mode in ('two', 'gates')
    rank1 = mode == 'rank1'
    wgt = torch.randn(cout, cin, k, k, device='cuda', generator=g) / (cin * k * k) ** 0.5
    bias = torch.randn(cout, device='cuda', generator=g)
    pc = ops.PackedConv(wgt, bias, 1, rank1_in=cin - 1 if rank1 else None, two_inputs=two,
                        precise=mode.startswith('precise'), act_lo8=mode.startswith('lo8'), gates=mode == 'gates',
                        nt_override=nt_override)
    x = torch.randn(b, h, w, pc.cin_pad, device='cuda', generator=g).half()
    kw, outs = {}, ('raw',)
    if two:
        kw['x2'] = torch.randn(b, h, w, pc.cin_pad, device='cuda', generator=g).half()
    if mode == 'gates':
        kw['gate_h'] = torch.randn(b, h, w, cout // 3, device='cuda', generator=g).half()
        outs = ('hidden',)
    if mode.startswith('precise'):
        kw['x_lo'] = (torch.randn(b, h, w, pc.cin_pad, device='cuda', generator=g) * 1e-3).half()
        outs = ('f32',) if mode == 'precise_splitk' else ('raw', 'raw_lo', 'relu', 'relu_lo')
    if mode.startswith('lo8'):
        kw['x_lo8'] = (torch.randn(b, h, w, pc.cin_pad, device='cuda', generator=g) * 4).to(torch.float8_e4m3fn) \
            .view(torch.uint8)
        outs = ('relu', 'relu_lo8') if mode == 'lo8' else ('raw', 'relu', 'relu_lo8')
    if mode in ('res', 'res_broadcast', 'lo8_res'):
        rb = 1 if mode == 'res_broadcast' else b
        kw['res'] = torch.randn(rb, h, w, cout, device='cuda', generator=g).half()
        kw['res_lo'] = (torch.randn(rb, h, w, cout, device='cuda', generator=g) * 1e-3).half()
        kw['res_broadcast'] = mode == 'res_broadcast'
        if mode == 'res':
            outs = ('raw', 'raw_lo', 'relu')
    if rank1:
        kw['rank1_x'] = torch.randn(b * h * w, device='cuda', generator=g)
        outs = ('raw', 'relu')
    if mode == 'relu':
        outs = ('relu',)
    if mode == 'head':
        kw['head_w'] = torch.randn(9, cout, device='cuda', generator=g)
        outs = ('relu',)
    if mode == 'f32':
        outs = ('raw', 'f32')
    return pc, x, kw, outs, (4 if mode == 'precise_splitk' else 0)


def _run(pc, x, kw, outs, ksplit, tile, nt, regs):
    from deva import _native as nat
    b, h, w, _ = x.shape
    ho, wo = pc.out_hw(h, w)
    n = b * ho * wo * pc.cout
    bufs = {}
    for name in outs:
        if name == 'relu_lo8':
            bufs[name] = torch.full((n + GUARD,), 0xFF, dtype=torch.uint8, device='cuda')  # 0xFF: e4m3 NaN
        elif name == 'f32':
            bufs[name] = torch.full((max(ksplit, 1) * n + GUARD,), float('nan'), device='cuda')
        elif name == 'hidden':
            bufs[name] = torch.full((n // 3 + GUARD,), float('nan'), dtype=torch.float16, device='cuda')
        else:
            bufs[name] = torch.full((n + GUARD,), float('nan'), dtype=torch.float16, device='cuda')
    head_w = kw.get('head_w')
    if head_w is not None:
        bufs['head'] = torch.full((b * ho * wo * head_w.shape[0] + GUARD,), float('nan'), device='cuda')
    old = os.environ.get('DEVA_B200_CONV_EPI')
    if regs:
        os.environ['DEVA_B200_CONV_EPI'] = 'regs'
    else:
        os.environ.pop('DEVA_B200_CONV_EPI', None)
    try:
        nat.conv2d(x, b, h, w, pc.cin_pad, pc.w_packed, pc.k, pc.stride, pc.cout, pc.cout_pad, nt, tile[0], tile[1],
                   pc.bias, x2=kw.get('x2'), x_lo=kw.get('x_lo'), res=kw.get('res'), res_lo=kw.get('res_lo'),
                   res_broadcast=kw.get('res_broadcast', False), rank1_w=pc.rank1_w, rank1_x=kw.get('rank1_x'),
                   out_raw=bufs.get('raw'), out_relu=bufs.get('relu'), out_f32=bufs.get('f32'),
                   out_raw_lo=bufs.get('raw_lo'), out_relu_lo=bufs.get('relu_lo'), head_w=head_w,
                   head_out=bufs.get('head'), head_n=0 if head_w is None else head_w.shape[0],
                   gate_h=kw.get('gate_h'), gate_out=bufs.get('hidden'), split_mode=pc.split_mode, ksplit=ksplit,
                   x_lo8=kw.get('x_lo8'), w8_packed=pc.w8_packed, acc_scale=pc.acc_scale,
                   out_relu_lo8=bufs.get('relu_lo8'))
    finally:
        if old is None:
            os.environ.pop('DEVA_B200_CONV_EPI', None)
        else:
            os.environ['DEVA_B200_CONV_EPI'] = old
    torch.cuda.synchronize()
    return bufs


_BITS = {torch.float16: torch.int16, torch.float32: torch.int32, torch.uint8: torch.uint8}


def _same(a, b, what):
    assert a.keys() == b.keys()
    for name in a:
        x, y = a[name].view(_BITS[a[name].dtype]), b[name].view(_BITS[b[name].dtype])
        diff = int((x != y).sum())
        assert diff == 0, f'{what}: {name} differs in {diff} of {x.numel()} elements'
        assert torch.equal(x[-GUARD:], y[-GUARD:]), f'{what}: {name} guard region written'


def _rect(ho, wo):
    from deva.model import native_ops as ops
    flat, ops.FLAT_TILES = ops.FLAT_TILES, False
    try:
        return ops.choose_tile(ho, wo)
    finally:
        ops.FLAT_TILES = flat


@pytest.mark.parametrize('regs', [False, True], ids=['own_epilogue', 'regs'])
@pytest.mark.parametrize('case', list(CASES))
def test_flat_tiles_match_rectangles(case, regs):
    from deva.model import native_ops as ops
    pc, x, kw, outs, ksplit = _inputs(case)
    ho, wo = pc.out_hw(x.shape[1], x.shape[2])
    assert ops.choose_tile(ho, wo) == ops.FLAT, (ho, wo)  # every case is a shape no rectangle fits
    flat = _run(pc, x, kw, outs, ksplit, ops.FLAT, pc.nt, regs)
    rect = _run(pc, x, kw, outs, ksplit, _rect(ho, wo), pc.nt, regs)
    _same(flat, rect, f'{case} flat vs rectangle')
    body = flat['hidden' if 'hidden' in flat else outs[0]][:-GUARD]
    assert not torch.isnan(body).any(), f'{case}: an output element was not written'


@pytest.mark.parametrize('regs', [False, True], ids=['staged', 'regs'])
@pytest.mark.parametrize('case,widths', [('3x3_b1_relu', (256, 128, 64)), ('act_lo8_b1', (256, 128)),
                                         ('ragged_res_broadcast', (256, 128, 64)), ('precise_1x1', (256, 128))])
def test_channel_tiles_match(case, widths, regs):
    """The same launch at each channel tile width, flat and rectangular pixel tiles: identical bits."""
    from deva.model import native_ops as ops
    pc, x, kw, outs, ksplit = _inputs(case)
    ho, wo = pc.out_hw(x.shape[1], x.shape[2])
    ref = _run(pc, x, kw, outs, ksplit, _rect(ho, wo), pc.nt, regs)
    for nt in widths:
        for tile in (ops.FLAT, _rect(ho, wo)):
            _same(_run(pc, x, kw, outs, ksplit, tile, nt, regs), ref, f'{case} nt {nt} tile {tile} vs nt {pc.nt}')


def test_flat_tiles_refuse_stride2_and_pool4():
    from deva import _native as nat
    from deva.model import native_ops as ops
    g = torch.Generator(device='cuda').manual_seed(0)
    pc = ops.PackedConv(torch.randn(64, 64, 3, 3, device='cuda', generator=g), None, 2)
    x = torch.randn(1, 68, 120, 64, device='cuda', generator=g).half()
    out = torch.empty(1, 34, 60, 64, dtype=torch.float16, device='cuda')
    with pytest.raises(RuntimeError, match='flat tiles'):
        nat.conv2d(x, 1, 68, 120, 64, pc.w_packed, 3, 2, 64, pc.cout_pad, pc.nt, 0, 128, pc.bias, out_raw=out)
    pc1 = ops.PackedConv(torch.randn(64, 64, 3, 3, device='cuda', generator=g), None, 1)
    pool = torch.empty(1, 17, 30, 64, dtype=torch.float16, device='cuda')
    with pytest.raises(RuntimeError, match='flat tiles'):
        nat.conv2d(x, 1, 68, 120, 64, pc1.w_packed, 3, 1, 64, pc1.cout_pad, pc1.nt, 0, 128, pc1.bias, out_pool4=pool)
