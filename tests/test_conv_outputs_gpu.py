"""Every output form of one convolution launch is derived from the same fp32 value, bit for bit.

One launch requests the fp32 result together with every fp16 / e4m3 form the epilogue can write: raw, ReLU'd, their
low-order parts and the e4m3 remainder of the ReLU'd value.  Each must equal the conversion of the fp32 output, on edge
tiles in both directions, on grids with more tiles than SMs, with an own or a batch-broadcast residual (hi, lo), with
and without the fused head, and on a ragged channel count that takes the element-by-element path.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

CASES = [
    # b, h, w, cin, cout, k, residual ('own' / 'broadcast' / None), fused head
    (2, 37, 45, 64, 256, 3, 'own', False),           # edge tiles in H and W
    (3, 100, 150, 128, 256, 3, 'own', True),         # more tiles than SMs, head as in up_8_4.out_conv.c2
    (4, 29, 61, 64, 256, 3, 'broadcast', False),     # the fuser's shared half: one residual image for the batch
    (2, 34, 50, 128, 512, 1, 'own', False),          # two channel tiles
    (3, 23, 41, 128, 192, 3, 'own', False),
    (2, 19, 27, 64, 129, 3, 'own', False),           # ragged Cout: element-by-element epilogue
    (2, 40, 72, 64, 256, 1, None, False),
]


def _lo8(v):  # e4m3 of (relu(v) - fp16(relu(v))) * 4096, as the next fp8 correction pass reads it
    a = v.clamp_min(0)
    return ((a - a.half().float()) * 4096).to(torch.float8_e4m3fn).float()


@pytest.mark.parametrize('b,h,w,cin,cout,k,res_kind,head', CASES)
def test_conv_outputs_are_conversions_of_the_fp32_result(b, h, w, cin, cout, k, res_kind, head):
    from deva import _native
    from deva.model import native_ops as ops
    _native.require_device()
    g = torch.Generator(device='cuda').manual_seed(b * 7919 + h * 31 + cout + k)
    x = torch.randn(b, h, w, cin, device='cuda', generator=g).half()
    wgt = torch.randn(cout, cin, k, k, device='cuda', generator=g) / (cin * k * k)**0.5
    bias = torch.randn(cout, device='cuda', generator=g)
    pc = ops.PackedConv(wgt, bias, 1)
    kw = {}
    if res_kind is not None:
        r = torch.randn(1 if res_kind == 'broadcast' else b, h, w, cout, device='cuda', generator=g)
        kw['res'] = r.half()
        kw['res_lo'] = (r - kw['res'].float()).half()
    if head:
        kw['head_w'] = torch.randn(9, cout, device='cuda', generator=g) / cout**0.5
    o = ops.conv_ex(x, pc, want_raw=True, want_relu=True, want_f32=True, want_lo=True, want_relu_lo8=True, **kw)
    torch.cuda.synchronize()
    v = o.f32
    assert torch.isfinite(v).all()
    raw = v.half()
    relu = v.clamp_min(0).half()
    assert torch.equal(o.raw, raw)
    assert torch.equal(o.raw_lo, (v - raw.float()).half())
    assert torch.equal(o.relu, relu)
    assert torch.equal(o.relu_lo, (v.clamp_min(0) - relu.float()).half())
    assert torch.equal(o.relu_lo8.view(torch.float8_e4m3fn).float(), _lo8(v))
    if res_kind is not None:  # the residual really was added: the fp32 result differs from the bare convolution
        bare = ops.conv_ex(x, pc, want_f32=True).f32
        want = bare + kw['res'].float() + kw['res_lo'].float()
        torch.cuda.synchronize()
        assert float((v - want).abs().max()) < 1e-5 * float(want.abs().max())
    if head:
        want = v.clamp_min(0).reshape(-1, cout).double() @ kw['head_w'].double().t()
        assert float((o.head.reshape(-1, 9).double() - want).abs().max()) < 1e-4 * float(want.abs().max())
