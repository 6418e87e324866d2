"""GPU parity of the NHWC fp16 network kernels against plain PyTorch fp32 ops on the same (fp16-rounded) inputs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ops():
    from deva import _native
    from deva.model import native_ops
    _native.require_device()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return native_ops


def _nhwc(x):  # fp32 NCHW -> fp16 NHWC
    return x.permute(0, 2, 3, 1).contiguous().half()


def _nchw(x):  # fp16/fp32 NHWC -> fp32 NCHW
    return x.float().permute(0, 3, 1, 2).contiguous()


CASES = [
    # b, h, w, cin, cout, k, stride
    (2, 20, 28, 64, 64, 3, 1),
    (1, 17, 23, 128, 256, 1, 1),
    (2, 20, 28, 64, 128, 3, 2),
    (1, 21, 27, 256, 512, 1, 2),
    (3, 9, 13, 512, 1536, 3, 1),
    (1, 30, 54, 1024, 512, 1, 1),
    (2, 16, 24, 256, 256, 3, 1),
    (1, 11, 19, 512, 129, 3, 1),   # key_proj-like ragged Cout (fp32 out)
    (2, 24, 40, 256, 1, 3, 1),     # pred-like single channel (fp32 out)
    # more tiles than SMs (132): several tiles per persistent CTA, the producer filling the ring for the next tile while
    # the consumers run the epilogue of the current one; odd tile counts leave a partial last wave
    (2, 136, 240, 128, 256, 3, 1),
    (5, 67, 119, 192, 320, 3, 1),
    (11, 100, 150, 128, 128, 3, 2),
    (5, 72, 121, 1024, 256, 1, 1),
    (3, 136, 241, 64, 256, 1, 1),
]


@pytest.mark.parametrize('b,h,w,cin,cout,k,stride', CASES)
def test_conv_matches_torch(b, h, w, cin, cout, k, stride):
    ops = _ops()
    g = torch.Generator(device='cuda').manual_seed(b * 1000 + cin + cout + k)
    x = torch.randn(b, cin, h, w, device='cuda', generator=g)
    wgt = torch.randn(cout, cin, k, k, device='cuda', generator=g) / (cin * k * k)**0.5
    bias = torch.randn(cout, device='cuda', generator=g)
    pc = ops.PackedConv(wgt, bias, stride)
    xh = _nhwc(x)
    ref = F.conv2d(xh.float().permute(0, 3, 1, 2), wgt.half().float(), bias, stride=stride, padding=k // 2)
    if cout % 8 == 0:
        ho, wo = ref.shape[-2:]
        res = torch.randn(b, cout, ho, wo, device='cuda', generator=g)
        raw, relu, f32 = ops.conv(xh, pc, res=_nhwc(res), want_raw=True, want_relu=True, want_f32=True)
        want = ref + _nhwc(res).float().permute(0, 3, 1, 2)
        torch.cuda.synchronize()
        assert float((_nchw(f32) - want).abs().max()) < 2e-3
        assert float((_nchw(raw) - want).abs().max()) < 1e-2
        assert float((_nchw(relu) - want.clamp_min(0)).abs().max()) < 1e-2
        # broadcast residual
        res1 = _nhwc(res[:1])
        f32b = ops.conv(xh, pc, res=res1, want_f32=True)
        wantb = ref + res1.float().permute(0, 3, 1, 2)
        torch.cuda.synchronize()
        assert float((_nchw(f32b) - wantb).abs().max()) < 2e-3
    else:
        f32 = ops.conv(xh, pc, want_f32=True)
        torch.cuda.synchronize()
        assert float((_nchw(f32) - ref).abs().max()) < 2e-3


@pytest.mark.parametrize('stride,k', [(1, 3), (2, 3), (2, 1)])
def test_conv_split_precision(stride, k):
    """x = hi + lo, W = hi + lo: D = Xh.Wh + Xl.Wh + Xh.Wl reproduces the fp32 convolution to ~1e-6 relative."""
    ops = _ops()
    g = torch.Generator(device='cuda').manual_seed(21 + stride + k)
    b, h, w, cin, cout = 2, 14, 18, 128, 256
    x = torch.randn(b, cin, h, w, device='cuda', generator=g)
    wgt = torch.randn(cout, cin, k, k, device='cuda', generator=g) / (cin * k * k)**0.5
    bias = torch.randn(cout, device='cuda', generator=g)
    pc = ops.PackedConv(wgt, bias, stride, precise=True)
    xh = _nhwc(x)
    xl = (x.permute(0, 2, 3, 1).contiguous() - xh.float()).half()
    ref = F.conv2d(x.double(), wgt.double(), bias.double(), stride=stride, padding=k // 2).float()
    res = torch.randn_like(ref)
    rh = _nhwc(res)
    rl = (res.permute(0, 2, 3, 1).contiguous() - rh.float()).half()
    o = ops.conv_ex(xh, pc, x_lo=xl, res=rh, res_lo=rl, want_raw=True, want_relu=True, want_f32=True, want_lo=True)
    torch.cuda.synchronize()
    want = ref + res
    scale = float(want.abs().max())
    assert float((_nchw(o.f32) - want).abs().max()) < 2e-5 * scale
    assert float((_nchw(o.raw) + _nchw(o.raw_lo) - want).abs().max()) < 2e-5 * scale
    assert float((_nchw(o.relu) + _nchw(o.relu_lo) - want.clamp_min(0)).abs().max()) < 2e-5 * scale
    # pooling on pairs
    y, y_lo = ops.maxpool(o.relu, o.relu_lo)
    wantp = F.max_pool2d(want.clamp_min(0), 3, 2, 1)
    assert float((_nchw(y) + _nchw(y_lo) - wantp).abs().max()) < 2e-5 * scale


def test_conv_fused_head_equals_3x3_conv():
    """c2 + residual, then pred(relu(.)) via the fused 9-tap head + gather == two separate convolutions."""
    ops = _ops()
    from deva import _native as nat
    g = torch.Generator(device='cuda').manual_seed(31)
    b, h, w, c = 2, 13, 22, 256
    x = torch.randn(b, c, h, w, device='cuda', generator=g)
    res = torch.randn(b, c, h, w, device='cuda', generator=g)
    wgt = torch.randn(c, c, 3, 3, device='cuda', generator=g) / (c * 9)**0.5
    bias = torch.randn(c, device='cuda', generator=g)
    pw = torch.randn(1, c, 3, 3, device='cuda', generator=g) / (c * 9)**0.5 * 3
    pb = 0.3
    pc = ops.PackedConv(wgt, bias, 1)
    head_w = pw[0].permute(1, 2, 0).reshape(9, c).contiguous()
    o = ops.conv_ex(_nhwc(x), pc, res=_nhwc(res), want_raw=True, head_w=head_w)
    logits = torch.empty(b, h, w, 1, device='cuda')
    nat.head_gather3x3(o.head, logits, pb, b, h, w)
    p4 = F.conv2d(_nhwc(x).float().permute(0, 3, 1, 2), wgt.half().float(), bias, padding=1) + _nhwc(res).float().permute(0, 3, 1, 2)
    ref = F.conv2d(F.relu(p4), pw, torch.tensor([pb], device='cuda'), padding=1)
    torch.cuda.synchronize()
    assert float((_nchw(o.raw) - p4).abs().max()) < 1e-2
    assert float((logits.permute(0, 3, 1, 2) - ref).abs().max()) < 2e-3


def test_conv_two_inputs():
    """GRU transform: conv3x3 over cat[g, h] without materialising the concat."""
    ops = _ops()
    g = torch.Generator(device='cuda').manual_seed(8)
    b, h, w, c, cout = 2, 9, 12, 512, 1536
    xa = torch.randn(b, c, h, w, device='cuda', generator=g)
    xb = torch.randn(b, c, h, w, device='cuda', generator=g)
    wgt = torch.randn(cout, 2 * c, 3, 3, device='cuda', generator=g) / (2 * c * 9)**0.5
    bias = torch.randn(cout, device='cuda', generator=g)
    pc = ops.PackedConv(wgt, bias, 1, two_inputs=True)
    out = ops.conv(_nhwc(xa), pc, x2=_nhwc(xb), want_f32=True)
    xin = torch.cat([_nhwc(xa).float().permute(0, 3, 1, 2), _nhwc(xb).float().permute(0, 3, 1, 2)], 1)
    ref = F.conv2d(xin, wgt.half().float(), bias, padding=1)
    torch.cuda.synchronize()
    assert float((_nchw(out) - ref).abs().max()) < 2e-3


@pytest.mark.parametrize('b,h,w', [(2, 9, 12), (16, 68, 60)])  # small: one tile per CTA; large: several
def test_conv_gate_epilogue(b, h, w):
    """Sensory update (modules.py:145-149): h' = f*h*(1-u) + u*tanh(n) from the fp32 accumulators of the 3x3 conv
    over cat[g, h]; the 3C-channel conv output is never written."""
    ops = _ops()
    g = torch.Generator(device='cuda').manual_seed(9)
    c = 512
    xg = torch.randn(b, c, h, w, device='cuda', generator=g)
    xh = torch.randn(b, c, h, w, device='cuda', generator=g)
    wgt = torch.randn(3 * c, 2 * c, 3, 3, device='cuda', generator=g) * (2.0 / (2 * c * 9))**0.5
    bias = torch.randn(3 * c, device='cuda', generator=g)
    pc = ops.PackedConv(wgt, bias, 1, two_inputs=True, gates=True)
    gh, hh = _nhwc(xg), _nhwc(xh)
    new_h = ops.conv_ex(gh, pc, x2=hh, gate_h=hh).hidden
    xin = torch.cat([gh.float().permute(0, 3, 1, 2), hh.float().permute(0, 3, 1, 2)], 1)
    v = F.conv2d(xin, wgt.half().float(), bias, padding=1)
    f, u, n = torch.sigmoid(v[:, :c]), torch.sigmoid(v[:, c:2 * c]), torch.tanh(v[:, 2 * c:])
    ref = f * hh.float().permute(0, 3, 1, 2) * (1 - u) + u * n
    torch.cuda.synchronize()
    assert float((_nchw(new_h) - ref).abs().max()) < 3e-3  # fp16 output rounding of |h'| <~ 4


def test_conv_rank1_term():
    ops = _ops()
    g = torch.Generator(device='cuda').manual_seed(5)
    b, h, w, cin, cout = 3, 10, 14, 513, 512
    x = torch.randn(b, cin, h, w, device='cuda', generator=g)
    wgt = torch.randn(cout, cin, 1, 1, device='cuda', generator=g) / cin**0.5
    bias = torch.randn(cout, device='cuda', generator=g)
    pc = ops.PackedConv(wgt, bias, 1, rank1_in=512)
    xh = _nhwc(x[:, :512])
    plane = x[:, 512].contiguous()
    out = ops.conv(xh, pc, rank1_x=plane, want_f32=True)
    wq = wgt.clone()
    wq[:, :512] = wq[:, :512].half().float()
    xin = torch.cat([xh.float().permute(0, 3, 1, 2), plane.unsqueeze(1)], 1)
    ref = F.conv2d(xin, wq, bias)
    torch.cuda.synchronize()
    assert float((_nchw(out) - ref).abs().max()) < 2e-3


@pytest.mark.parametrize('k_obj,h,w', [(1, 32, 48), (3, 48, 80), (2, 44, 520)])  # last: ragged row group / column block
def test_stem_matches_torch(k_obj, h, w):
    """7x7 s2 stem = shared image part (3 ch) + per-object mask part (1 ch), both through im2col + 1x1 GEMM."""
    ops = _ops()
    g = torch.Generator(device='cuda').manual_seed(11)
    image = torch.randn(1, 3, h, w, device='cuda', generator=g)
    masks = torch.rand(k_obj, 1, h, w, device='cuda', generator=g)
    wgt = torch.randn(64, 4, 7, 7, device='cuda', generator=g) / (4 * 49)**0.5
    bias = torch.randn(64, device='cuda', generator=g) * 0.1
    pc_img = ops.pack_stem(wgt[:, :3], bias)
    pc_msk = ops.pack_stem(wgt[:, 3:], None)
    shared = ops.conv(ops.stem_columns(image, pc_img.cin_pad), pc_img, want_raw=True)
    out = ops.conv(ops.stem_columns(masks, pc_msk.cin_pad), pc_msk, res=shared, want_relu=True)
    xin = torch.cat([image.half().float().expand(k_obj, -1, -1, -1), masks.half().float()], 1)
    ref = F.relu(F.conv2d(xin, wgt.half().float(), bias, stride=2, padding=3))
    torch.cuda.synchronize()
    assert float((_nchw(out) - ref).abs().max()) < 1e-2


@pytest.mark.parametrize('c,h,w,with_lo', [(1, 44, 520, False), (3, 44, 520, True), (3, 32, 48, False), (2, 20, 36, True)])
def test_stem_columns_exact(c, h, w, with_lo):
    """im2col of the 7x7 stride-2 pad-3 stems: column (ky*7 + kx)*C + c, fp16 value and fp16 remainder, zero padded -
    bit-exact against F.unfold for the pixel-per-thread kernels (C = 1, 3) and the generic one (C = 2)."""
    ops = _ops()
    g = torch.Generator(device='cuda').manual_seed(5)
    x = torch.randn(2, c, h, w, device='cuda', generator=g)
    kp = (49 * c + 63) // 64 * 64
    got = ops.stem_columns(x, kp, with_lo=with_lo)
    cols = F.unfold(x, 7, padding=3, stride=2).view(2, c, 49, h // 2, w // 2)   # [B, c, tap, Ho, Wo]
    ref = torch.zeros(2, h // 2, w // 2, kp, device='cuda')
    ref[..., :49 * c] = cols.permute(0, 3, 4, 2, 1).reshape(2, h // 2, w // 2, 49 * c)
    hi = got[0] if with_lo else got
    torch.cuda.synchronize()
    assert torch.equal(hi, ref.half())
    if with_lo:
        assert torch.equal(got[1], (ref - ref.half().float()).half())


def test_helpers_match_torch():
    ops = _ops()
    from deva import _native as nat
    g = torch.Generator(device='cuda').manual_seed(3)
    x = torch.randn(2, 64, 18, 26, device='cuda', generator=g)
    xh = _nhwc(x)
    xf = xh.float().permute(0, 3, 1, 2)
    torch.testing.assert_close(_nchw(ops.maxpool(xh)), F.max_pool2d(xf, 3, 2, 1))
    y = torch.randn(2, 64, 16, 24, device='cuda', generator=g)
    yh = _nhwc(y)
    for r in (2, 4):
        want = F.interpolate(yh.float().permute(0, 3, 1, 2), scale_factor=1 / r, mode='area')
        assert float((_nchw(ops.area_down(yh, r)) - want).abs().max()) < 2e-3
    plane = torch.rand(3, 32, 48, device='cuda', generator=g)
    torch.testing.assert_close(ops.area_down_plane(plane, 16), F.interpolate(plane.unsqueeze(0), size=(2, 3), mode='area')[0])
    # output tail
    k, hq, wq = 3, 6, 10
    logits = torch.randn(k, hq, wq, device='cuda', generator=g) * 3
    agg = torch.empty(k + 1, hq, wq, device='cuda')
    prob = torch.empty(k + 1, 4 * hq, 4 * wq, device='cuda')
    lo = torch.empty_like(prob)
    nat.output_tail(logits, agg, prob, lo, k, hq, wq)
    pr = torch.sigmoid(logits)
    full = torch.cat([torch.prod(1 - pr, 0, keepdim=True), pr], 0).clamp(1e-7, 1 - 1e-7)
    ref_l = F.interpolate(torch.log(full / (1 - full)).unsqueeze(0), scale_factor=4, mode='bilinear', align_corners=False)[0]
    torch.cuda.synchronize()
    assert float((lo - ref_l).abs().max()) < 1e-4
    assert float((prob - torch.softmax(ref_l, 0)).abs().max()) < 1e-5
    # key tail
    q, ck = 37, 64
    yk = torch.randn(q, 160, device='cuda', generator=g)
    key, shr, sel = torch.empty(q, ck, device='cuda'), torch.empty(q, device='cuda'), torch.empty(q, ck, device='cuda')
    nat.key_tail(yk, 160, q, ck, key, shr, sel)
    torch.cuda.synchronize()
    assert torch.equal(key, yk[:, :ck])
    torch.testing.assert_close(shr, yk[:, ck]**2 + 1)
    torch.testing.assert_close(sel, torch.sigmoid(yk[:, ck + 1:2 * ck + 1]))
    # transpose append
    src = torch.randn(70, 96, device='cuda', generator=g).half()
    dst = torch.zeros(96, 128, dtype=torch.float16, device='cuda')
    nat.transpose_append(src, dst[:, 8:], 128, 70, 96)
    torch.cuda.synchronize()
    assert torch.equal(dst[:, 8:78], src.t())
    # layout converter: fp32 NCHW -> fp16 NHWC, channels 5..7 zero padding
    img = torch.randn(2, 5, 7, 9, device='cuda', generator=g)
    d = torch.full((2, 7, 9, 8), float('nan'), dtype=torch.float16, device='cuda')
    nat.nchw_to_nhwc(img, d, 2, 5, 7, 9, 8)
    torch.cuda.synchronize()
    assert torch.equal(d[..., :5], img.half().permute(0, 2, 3, 1)) and bool((d[..., 5:] == 0).all())
