"""GPU probe: how accurate is the split-precision (3-pass fp16 hi/lo) convolution, and is the residual error the tensor
core's fp32 accumulation?  Compares one deep-K conv against fp64, whole and as a sum of K-chunks added in fp32 on the
CUDA cores (if the chunked sum is markedly better, in-register accumulation is what limits the key path)."""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tracking-anything-with-deva_b200'))
from deva.model import native_ops as ops  # noqa: E402

torch.set_grad_enabled(False)


def split(x):
    hi = x.half()
    return hi, (x - hi.float()).half()


def main():
    g = torch.Generator(device='cuda').manual_seed(0)
    for (cin, k, relu_in) in ((256, 3, True), (1024, 1, True), (512, 3, False), (2048, 1, True)):
        b, h, w, cout = 2, 24, 40, 256
        x = torch.randn(b, cin, h, w, device='cuda', generator=g)
        if relu_in:
            x = x.relu()
        wgt = torch.randn(cout, cin, k, k, device='cuda', generator=g) / (cin * k * k) ** 0.5
        ref = F.conv2d(x.double(), wgt.double(), padding=k // 2)
        scale = float(ref.abs().max())
        xh, xl = split(x.permute(0, 2, 3, 1).contiguous())
        full = ops.conv_ex(xh, ops.PackedConv(wgt, None, 1, precise=True), x_lo=xl, want_f32=True).f32.permute(0, 3, 1, 2).double()
        parts = 0
        for c0 in range(0, cin, 64):
            pc = ops.PackedConv(wgt[:, c0:c0 + 64].contiguous(), None, 1, precise=True)
            parts = parts + ops.conv_ex(xh[..., c0:c0 + 64].contiguous(), pc, x_lo=xl[..., c0:c0 + 64].contiguous(),
                                        want_f32=True).f32.permute(0, 3, 1, 2).float()
        f32 = F.conv2d(x, wgt, padding=k // 2).double()
        torch.cuda.synchronize()
        for name, got in (('3-pass, one accumulator', full), ('3-pass, 64-ch chunks summed in fp32', parts.double()),
                          ('cuDNN fp32 (no TF32)', f32)):
            d = got - ref
            print(f'cin {cin:5d} k {k} relu_in {int(relu_in)}  {name:40s} max {float(d.abs().max()) / scale:.2e}  '
                  f'rms {float(d.pow(2).mean().sqrt()) / scale:.2e}  mean signed {float(d.mean()) / scale:+.2e}  '
                  f'mean signed on |ref|-weighted {float((d * ref.sign()).mean()) / scale:+.2e}')


if __name__ == '__main__':
    torch.backends.cudnn.allow_tf32 = False
    main()
