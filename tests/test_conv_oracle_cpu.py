"""oracle/conv_desc.py, the float64 semantics of one convolution launch, against float64 F.conv2d on the unpacked
weights.  The operands are packed by native_ops.PackedConv on the CPU in every mode it has (plain, two inputs, split
precision, weight hi/lo, the fp8 correction pass, rank-1 input, gates, the stem, ragged Cout, cin_pad > cin), so the
oracle's reading of the packed layout, the pass list, the k-iteration numbering and the chain boundaries of split-K are
pinned independently of the kernel it judges."""
import pytest
import torch
import torch.nn.functional as F

from oracle import conv_desc as cd

TOL = 1e-12  # of max |reference|: float64 rounding only


def _ops():
    from deva.model import native_ops
    return native_ops


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _nhwc(x, cin_pad):
    """fp32 [B, C, H, W] -> fp16 NHWC [B, H, W, cin_pad], zero padded."""
    b, c, h, w = x.shape
    out = torch.zeros(b, h, w, cin_pad, dtype=torch.float16)
    out[..., :c] = x.permute(0, 2, 3, 1).half()
    return out


def _desc(pc, x, **kw):
    b, h, w, _ = x.shape
    ho, wo = pc.out_hw(h, w)
    d = dict(x=x, batch=b, h=h, w=w, cin_pad=pc.cin_pad, w_packed=pc.w_packed, kh=pc.k, stride=pc.stride, cout=pc.cout,
             cout_pad=pc.cout_pad, nt=pc.nt, th=1, tw=128, bias=pc.bias, rank1_w=pc.rank1_w, split_mode=pc.split_mode,
             w8_packed=pc.w8_packed, acc_scale=pc.acc_scale, out_f32=torch.empty(0))
    d.update(kw)
    return d, ho, wo


def _as_nchw(v, b, ho, wo):
    return v.view(b, ho, wo, -1).permute(0, 3, 1, 2)


def _close(got, ref, what):
    err = float((got - ref).abs().max()) / max(float(ref.abs().max()), 1e-300)
    assert err <= TOL, f'{what}: {err:.2e}'


def _w16(shape, g, scale=1.0):
    """fp32 weights exactly representable in fp16 (plain packing is then lossless)."""
    return (torch.randn(*shape, generator=g) * scale).half().float()


@pytest.mark.parametrize('k,stride,cin,cout,h,w', [
    (3, 1, 64, 64, 9, 11), (1, 1, 128, 256, 5, 7), (3, 2, 64, 33, 9, 13), (3, 2, 65, 129, 8, 5),
    (1, 2, 64, 1, 7, 7), (3, 1, 100, 200, 1, 1), (3, 2, 64, 64, 1, 6)])
def test_plain_matches_conv2d(k, stride, cin, cout, h, w):
    """Plain packing with ragged Cout, cin_pad > cin, stride 2 on odd sides, 1-pixel images."""
    ops = _ops()
    g = _g(k * 1000 + cout + h)
    b = 2
    wgt, bias = _w16((cout, cin, k, k), g), torch.randn(cout, generator=g)
    x = torch.randn(b, cin, h, w, generator=g).half().float()
    pc = ops.PackedConv(wgt, bias, stride)
    assert (cin % 64 != 0) == (pc.cin_pad > cin)
    d, ho, wo = _desc(pc, _nhwc(x, pc.cin_pad))
    o = cd.launch(**d)
    ref = F.conv2d(x.double(), wgt.double(), bias.double(), stride=stride, padding=k // 2)
    assert ref.shape[-2:] == (ho, wo)
    _close(_as_nchw(o.value, b, ho, wo), ref, 'plain')
    assert o.nk == [k * k * pc.cin_pad // 64] and len(o.chains) == 1
    assert bool((o.mag >= o.value.abs() * (1 - 1e-12)).all())
    # a pixel subset gives the same rows
    sub = torch.tensor([0, b * ho * wo - 1, ho * wo // 2])
    _close(cd.launch(pixels=sub, **d).value, o.value[sub], 'pixel subset')


def test_two_inputs_rank1_and_residuals():
    """x2 (implicit concat), the rank-1 input channel, an own and a broadcast residual with its low-order part."""
    ops = _ops()
    g = _g(5)
    b, h, w, c, cout = 3, 6, 7, 128, 64
    wgt, bias = _w16((cout, 2 * c, 3, 3), g), torch.randn(cout, generator=g)
    x = torch.randn(b, 2 * c, h, w, generator=g).half().float()
    pc = ops.PackedConv(wgt, bias, 1, two_inputs=True)
    d, ho, wo = _desc(pc, _nhwc(x[:, :c], c), x2=_nhwc(x[:, c:], c))
    ref = F.conv2d(x.double(), wgt.double(), bias.double(), padding=1)
    _close(_as_nchw(cd.launch(**d).value, b, ho, wo), ref, 'two inputs')

    cin = 65  # the rank-1 channel is the last: 64 channels stay, cin_pad 64
    wgt, bias = _w16((cout, cin, 1, 1), g), torch.randn(cout, generator=g)
    x = torch.randn(b, cin, h, w, generator=g).half().float()
    pc = ops.PackedConv(wgt, bias, 1, rank1_in=cin - 1)
    res = torch.randn(b, h, w, cout, generator=g).half()
    res_lo = (torch.randn(b, h, w, cout, generator=g) * 1e-3).half()
    plane = x[:, cin - 1].contiguous().view(-1)
    ref = F.conv2d(x.double(), wgt.double(), bias.double())
    for rb in (b, 1):
        d, ho, wo = _desc(pc, _nhwc(x[:, :cin - 1], 64), rank1_x=plane, res=res[:rb], res_lo=res_lo[:rb],
                          res_broadcast=rb == 1, out_raw=torch.empty(0))
        o = cd.launch(**d)
        want = ref + (res[:rb].double() + res_lo[:rb].double()).permute(0, 3, 1, 2)
        _close(_as_nchw(o.value, b, ho, wo), want, f'rank-1 + residual (batch {rb})')
        assert torch.equal(o.outputs['raw'], o.value.float().half())


@pytest.mark.parametrize('mode', ['precise', 'w_lo', 'act_lo8'])
def test_split_precision_modes(mode):
    """(hi, lo) passes: Xh.Wh + Xl.Wh + Xh.Wl, X.Wh + X.Wl; the fp8 pass (X.W16 + Xlo8.W8) * 2^-S."""
    ops = _ops()
    g = _g(len(mode))
    b, cin, cout, h, w, k = 2, 128, 96, 5, 6, 3
    wgt, bias = torch.randn(cout, cin, k, k, generator=g) / 30, torch.randn(cout, generator=g)
    pc = ops.PackedConv(wgt, bias, 1, precise=mode == 'precise', w_lo=mode == 'w_lo', act_lo8=mode == 'act_lo8')
    x = torch.randn(b, cin, h, w, generator=g)
    xh = x.half().float()
    conv = lambda a, wt: F.conv2d(a.double(), wt.double(), padding=1)  # noqa: E731
    wh = wgt.half().float()
    wl = (wgt - wh).half().float()
    kw = {}
    if mode == 'precise':
        xl = (x - xh).half().float()
        kw['x_lo'] = _nhwc(xl, cin)
        ref = conv(xh, wh) + conv(xl, wh) + conv(xh, wl)
    elif mode == 'w_lo':
        ref = conv(xh, wh) + conv(xh, wl)
    else:
        s = -round(torch.log2(torch.tensor(pc.acc_scale)).item())
        assert pc.acc_scale == 2.0 ** -s
        lo8 = ((x - xh) * 4096).to(torch.float8_e4m3fn)
        kw['x_lo8'] = lo8.permute(0, 2, 3, 1).contiguous().view(torch.uint8)
        w8 = (wgt * 2.0 ** (s - 12)).to(torch.float8_e4m3fn).float()
        ref = (conv(xh, (wgt * 2.0 ** s).half().float()) + conv(lo8.float(), w8)) * 2.0 ** -s
        assert float((ref - conv(x, wgt)).abs().max()) < 2e-3 * float(ref.abs().max())  # what the pass is for
    ref = ref + bias.double().view(1, -1, 1, 1)
    d, ho, wo = _desc(pc, _nhwc(xh, cin), **kw)
    o = cd.launch(**d)
    _close(_as_nchw(o.value, b, ho, wo), ref, mode)
    n16 = 9 * 2 * (3 if mode == 'precise' else 2 if mode == 'w_lo' else 1)
    assert o.k8 == (9 if mode == 'act_lo8' else 0) and o.k_iters == n16 + o.k8


def test_gates_regrouping():
    """Gate rows regrouped into [f | u | n] x 64 tiles: the oracle's gate output equals the update computed on the
    reference convolution's unpermuted channels."""
    ops = _ops()
    g = _g(11)
    b, c, hid, h, w = 2, 64, 128, 5, 4
    wgt, bias = _w16((3 * hid, 2 * c, 3, 3), g, 0.05), torch.randn(3 * hid, generator=g)
    x = torch.randn(b, 2 * c, h, w, generator=g).half().float()
    hprev = torch.randn(b, h, w, hid, generator=g).half()
    pc = ops.PackedConv(wgt, bias, 1, two_inputs=True, gates=True)
    assert pc.nt == 192 and pc.cout_pad == 3 * hid
    d, ho, wo = _desc(pc, _nhwc(x[:, :c], c), x2=_nhwc(x[:, c:], c), gate_h=hprev, gate_out=torch.empty(0))
    d.pop('out_f32')
    o = cd.launch(**d)
    ref = F.conv2d(x.double(), wgt.double(), bias.double(), padding=1).permute(0, 2, 3, 1).reshape(-1, 3 * hid)
    f, u, n = torch.sigmoid(ref[:, :hid]), torch.sigmoid(ref[:, hid:2 * hid]), torch.tanh(ref[:, 2 * hid:])
    want = f * hprev.double().view(-1, hid) * (1 - u) + u * n
    _close(o.outputs['gate'], want, 'gates')


def test_stem_packing():
    """pack_stem: the 7x7 stride-2 stem as a 1x1 conv over (kh, kw, c) im2col columns."""
    ops = _ops()
    g = _g(3)
    b, h, w = 1, 16, 22
    wgt, bias = _w16((64, 3, 7, 7), g, 0.1), torch.randn(64, generator=g)
    x = torch.randn(b, 3, h, w, generator=g).half().float()
    pc = ops.pack_stem(wgt, bias)
    cols = F.unfold(x, 7, padding=3, stride=2).view(b, 3, 7, 7, h // 2, w // 2).permute(0, 4, 5, 2, 3, 1)
    xc = torch.zeros(b, h // 2, w // 2, pc.cin_pad, dtype=torch.float16)
    xc[..., :147] = cols.reshape(b, h // 2, w // 2, 147).half()
    d, ho, wo = _desc(pc, xc)
    ref = F.conv2d(x.double(), wgt.double(), bias.double(), stride=2, padding=3)
    _close(_as_nchw(cd.launch(**d).value, b, ho, wo), ref, 'stem')


def test_head_and_pool4():
    ops = _ops()
    g = _g(17)
    b, cin, cout, h, w = 2, 64, 64, 8, 12
    wgt, bias = _w16((cout, cin, 3, 3), g), torch.randn(cout, generator=g)
    x = torch.randn(b, cin, h, w, generator=g).half().float()
    pc = ops.PackedConv(wgt, bias, 1)
    head_w = torch.randn(9, cout, generator=g)
    d, ho, wo = _desc(pc, _nhwc(x, cin), head_w=head_w, head_n=9, head_out=torch.empty(0), out_pool4=torch.empty(0))
    d.pop('out_f32')
    o = cd.launch(**d)
    ref = F.conv2d(x.double(), wgt.double(), bias.double(), padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
    _close(o.outputs['head'], ref.clamp_min(0) @ head_w.double().t(), 'head')
    raw = ref.float().half().double().view(b, ho // 4, 4, wo // 4, 4, cout).mean((2, 4)).half().view(-1, cout)
    assert torch.equal(o.outputs['pool4'], raw) and torch.equal(o.outputs['pool4_win'], torch.arange(raw.shape[0]))
    # a subset holding whole windows only pools those
    sub = torch.tensor([y * wo + x for y in range(4) for x in range(4, 8)] + [0, 1])
    s = cd.launch(pixels=sub, **d)
    assert s.outputs['pool4_win'].tolist() == [1] and torch.equal(s.outputs['pool4'], raw[1:2])


@pytest.mark.parametrize('stride,cin,ksplit,n_parts', [
    (1, 512, 4, 4), (1, 512, 5, 5), (1, 512, 7, 7), (1, 128, 10, 9), (2, 128, 20, 18), (2, 256, 8, 8)])
def test_split_k_chains(stride, cin, ksplit, n_parts):
    """Chains sum to the whole value, their count is test_precision_gpu.py::test_conv_split_k_partial_sums's (54
    k-iterations at ksplit 10 -> chains of 6 -> 9 parts), only chain 0 has the bias, and each chain is the sum of its own
    k-iterations (pass, tap, 64-channel block) computed one by one from the unpacked weights."""
    ops = _ops()
    g = _g(cin + ksplit)
    b, h, w, cout = 1, 5, 7, 129
    wgt, bias = torch.randn(cout, cin, 3, 3, generator=g) / 40, torch.randn(cout, generator=g)
    pc = ops.PackedConv(wgt, bias, stride, precise=True)
    x = torch.randn(b, cin, h, w, generator=g)
    xh = x.half().float()
    xl = (x - xh).half().float()
    d, ho, wo = _desc(pc, _nhwc(xh, cin), x_lo=_nhwc(xl, cin), ksplit=ksplit)
    o = cd.launch(**d)
    whole = cd.launch(**dict(d, ksplit=0))
    assert len(o.chains) == n_parts and o.outputs['f32'].shape[0] == n_parts
    _close(o.value, whole.value, 'sum of chains')
    wh = wgt.half().float()
    wl = (wgt - wh).half().float()
    passes = [(xh, wh), (xl, wh), (xh, wl)]
    cb = cin // 64
    for c, (k0, k1) in enumerate(o.chains):
        want = torch.zeros(b, cout, ho, wo, dtype=torch.float64)
        for ki in range(k0, k1):
            t, blk = divmod(ki, cb)
            (xs, ws), tap = passes[t // 9], t % 9
            mask = torch.zeros_like(ws)
            mask[:, 64 * blk:64 * (blk + 1), tap // 3, tap % 3] = 1
            want += F.conv2d(xs.double(), (ws * mask).double(), stride=stride, padding=1)
        if c == 0:
            want += bias.double().view(1, -1, 1, 1)
        _close(_as_nchw(o.chain_value[c], b, ho, wo), want, f'chain {c} [{k0}, {k1})')


def test_refuses_what_the_kernel_refuses():
    ops = _ops()
    pc = ops.PackedConv(torch.randn(576, 128, 3, 3), None, 1, two_inputs=True, gates=True)
    x = torch.zeros(1, 4, 4, 64, dtype=torch.float16)
    d, _, _ = _desc(pc, x, x2=x, gate_h=torch.zeros(1, 4, 4, 192, dtype=torch.float16), gate_out=torch.empty(0),
                    acc_scale=0.5)
    with pytest.raises(ValueError, match='gate'):
        cd.launch(**d)
    with pytest.raises(ValueError, match='exclusive'):
        cd.launch(**dict(d, x_lo=x, acc_scale=0.0))
    with pytest.raises(ValueError, match='ksplit'):
        cd.launch(**dict(d, gate_out=None, ksplit=1000, acc_scale=0.0))
