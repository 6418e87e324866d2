"""The fused logit head at every channel width it admits, and its refusal of a channel count it does not.

The head epilogue runs only the full-width column loop, so it accepts a layer whose whole Cout is one channel tile of
exactly 64, 128, 192 or 256 channels.  Each width is its own kernel instantiation; the network's head (Cout 256) is
also covered by test_conv_outputs_gpu.py.  Edge tiles in H and W leave some rows of a tile outside the image.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ops():
    from deva import _native
    from deva.model import native_ops
    _native.require_device()
    return native_ops


@pytest.mark.parametrize('cout,head_n', [(64, 9), (128, 4), (192, 1)])
def test_fused_head_matches_float64(cout, head_n):
    ops = _ops()
    b, h, w, cin = 2, 37, 45, 128
    g = torch.Generator(device='cuda').manual_seed(cout + head_n)
    x = torch.randn(b, h, w, cin, device='cuda', generator=g).half()
    wgt = torch.randn(cout, cin, 3, 3, device='cuda', generator=g) / (cin * 9)**0.5
    bias = torch.randn(cout, device='cuda', generator=g)
    pc = ops.PackedConv(wgt, bias, 1)
    r = torch.randn(b, h, w, cout, device='cuda', generator=g)
    res = r.half()
    res_lo = (r - res.float()).half()
    head_w = torch.randn(head_n, cout, device='cuda', generator=g) / cout**0.5
    o = ops.conv_ex(x, pc, res=res, res_lo=res_lo, want_raw=True, want_f32=True, head_w=head_w)
    torch.cuda.synchronize()
    v = o.f32
    assert torch.isfinite(v).all()
    assert torch.equal(o.raw, v.half())
    want = v.clamp_min(0).reshape(-1, cout).double() @ head_w.double().t()
    assert float((o.head.reshape(-1, head_n).double() - want).abs().max()) < 1e-4 * float(want.abs().max())


def test_fused_head_rejects_a_ragged_channel_count():
    ops = _ops()
    b, h, w, cin, cout = 1, 16, 16, 64, 96  # one 96-wide channel tile: no full-width head loop for it
    g = torch.Generator(device='cuda').manual_seed(96)
    x = torch.randn(b, h, w, cin, device='cuda', generator=g).half()
    pc = ops.PackedConv(torch.randn(cout, cin, 3, 3, device='cuda', generator=g), None, 1)
    head_w = torch.randn(9, cout, device='cuda', generator=g)
    with pytest.raises(RuntimeError, match='fused head'):
        ops.conv_ex(x, pc, want_raw=True, head_w=head_w)
