"""Micro-benchmark of deva_b200_conv2d on the decoder's dominant layer shapes (C3: 16 objects, 1080p)."""
import argparse, json, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tracking-anything-with-deva_b200'))
from deva import _native as nat  # noqa: E402
from deva.model import native_ops as ops  # noqa: E402

CASES = {
    # name: (batch, h, w, cin, cout, k, mode)
    'up84_c1': (16, 272, 480, 256, 256, 3, 'relu'),
    # what up_8_4.out_conv.c1 runs in the parity plan: an e4m3 correction pass over the low-order activations, then the
    # fp16 pass, writing the ReLU'd output and its e4m3 low-order part for the next layer
    'up84_c1_lo8': (16, 272, 480, 256, 256, 3, 'actlo8'),
    # what up_8_4.out_conv.c2 runs in the parity plan: the e4m3 correction pass, the residual as (hi, lo) and the fused head
    'up84_c2_parity': (16, 272, 480, 256, 256, 3, 'actlo8+res+head'),
    # the same launch without the head: the difference to up84_c2_parity is what the fused head costs
    'up84_c2_parity_nohead': (16, 272, 480, 256, 256, 3, 'actlo8+res'),
    'up84_c2_res': (16, 272, 480, 256, 256, 3, 'raw+res'),
    'up84_c2_head': (16, 272, 480, 256, 256, 3, 'raw+res+head'),
    'gru': (16, 68, 120, 512, 1536, 3, 'two'),
    'fuser_c2': (16, 68, 120, 512, 512, 3, 'raw+res'),
    'up168_c1': (16, 136, 240, 512, 256, 3, 'relu'),
    'ds_1x1': (16, 136, 240, 512, 256, 1, 'raw'),
    'res2_c3_precise': (1, 272, 480, 64, 256, 1, 'precise'),
    # shallow-K layers (epilogue / latency bound): sensory updater 1x1 convs, the mask stem as a 1x1 GEMM over 64 im2col columns
    'g16_1x1': (16, 68, 120, 512, 512, 1, 'raw'),
    'g8_1x1_res': (16, 68, 120, 256, 512, 1, 'raw+res'),
    'stem_1x1': (16, 544, 960, 64, 64, 1, 'relu'),
    # the sensory update as the product runs it: gate epilogue, 192-column tiles; and the plain epilogue on 192-column tiles
    'gru_gates': (16, 68, 120, 512, 1536, 3, 'gates'),
    'gru_n192': (16, 68, 120, 512, 1536, 3, 'two192'),
    # batch-1 layers at 1/16 (the pixel encoder's layer3, the projections, the fusers' shared halves): 64 flat pixel
    # tiles, so the channel tile decides how many SMs they occupy
    'layer3_c2_precise_b1': (1, 68, 120, 256, 256, 3, 'precise'),
    'proj1_b1': (1, 68, 120, 1024, 512, 1, 'raw'),
    'fuser_c1x_b1': (1, 68, 120, 512, 512, 3, 'raw'),
}


def run(name, iters=8):
    b, h, w, cin, cout, k, mode = CASES[name]
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(b, h, w, cin, device=dev, generator=g).half()
    two = mode in ('two', 'gates', 'two192')
    wgt = torch.randn(cout, cin * (2 if two else 1), k, k, device=dev, generator=g) / (cin * k * k)**0.5
    bias = torch.randn(cout, device=dev, generator=g)
    pc = ops.PackedConv(wgt, bias, 1, two_inputs=two, precise=(mode == 'precise'), act_lo8=mode.startswith('actlo8'),
                        gates=(mode == 'gates'), nt_override=192 if mode == 'two192' else None)
    kw = {}
    if two:
        kw['x2'] = torch.randn_like(x)
    if mode == 'gates':
        kw['gate_h'] = kw['x2']
    if mode == 'precise':
        kw['x_lo'] = (torch.randn_like(x) * 1e-3)
    if mode.startswith('actlo8'):  # e4m3 of (x - fp16(x)) * 4096
        kw['x_lo8'] = (torch.randn_like(x, dtype=torch.float32) * 4).to(torch.float8_e4m3fn).view(torch.uint8)
    if 'res' in mode:
        kw['res'] = torch.randn(b, h, w, cout, device=dev, generator=g).half()
        if mode.startswith('actlo8'):
            kw['res_lo'] = (torch.randn(b, h, w, cout, device=dev, generator=g) * 1e-3).half()
    if 'head' in mode:
        kw['head_w'] = torch.randn(9, cout, device=dev, generator=g)
    want = dict(want_relu=True) if mode in ('relu', ) else (dict() if mode == 'gates' else dict(want_raw=True))
    if mode == 'precise':
        want = dict(want_relu=True, want_lo=True)
    if mode == 'actlo8':
        want = dict(want_relu=True, want_relu_lo8=True)
    # fp16-equivalent MMA passes; the e4m3 pass does the same MACs at twice the rate, so it counts as half a pass
    passes = 3 if mode == 'precise' else (2 if two else (1.5 if mode.startswith('actlo8') else 1))
    flops = 2.0 * b * h * w * cout * k * k * pc.cin_pad * passes
    for _ in range(3):
        ops.conv_ex(x, pc, **kw, **want)
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); ops.conv_ex(x, pc, **kw, **want); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    ms = ts[len(ts) // 2]
    return dict(case=name, ms=ms, tflops=flops / ms / 1e9, gflop=flops / 1e9)


# The measured fp16 tensor-core ceiling on the card at hand: cuBLAS on one GEMM with the N and K of up84_c1 (Cout 256,
# 3x3 x 256 channels) and M = 8 waves of 128-row tiles on 132 SMs.
MATMULS = {'cublas_up84': (132 * 128 * 8, 256, 9 * 256)}


def run_matmul(name, iters=8, reps=10):
    m, n, k = MATMULS[name]
    g = torch.Generator(device='cuda').manual_seed(0)
    a = torch.randn(m, k, device='cuda', generator=g).half()
    b = torch.randn(k, n, device='cuda', generator=g).half()
    for _ in range(3):
        torch.matmul(a, b)
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            torch.matmul(a, b)
        e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / reps)
    ts.sort()
    ms = ts[len(ts) // 2]
    flops = 2.0 * m * n * k
    return dict(case=name, ms=ms, tflops=flops / ms / 1e9, gflop=flops / 1e9)


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--cases', default=','.join([*CASES, *MATMULS]))
    ap.add_argument('--rect', action='store_true', help='rectangular pixel tiles only (no flat tiles at 1/16)')
    ap.add_argument('--packed-nt', action='store_true', help='every launch takes the packed channel tile')
    a = ap.parse_args()
    nat.require_device()
    if a.rect:
        ops.FLAT_TILES = False
    if a.packed_nt:
        ops.choose_nt = lambda nt, *_: nt
    for c in a.cases.split(','):
        print(json.dumps(run_matmul(c) if c in MATMULS else run(c)))
