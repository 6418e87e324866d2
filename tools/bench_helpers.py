"""Achieved HBM GB/s of the memory-bound helper kernels at C3 shapes (CUDA events, median of 10)."""
import json, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tracking-anything-with-deva_b200'))
from deva import _native as nat  # noqa: E402
from deva.model import native_ops as ops  # noqa: E402


def timeit(fn, iters=10):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    nat.require_device()
    dev = 'cuda'
    K, h, w = 16, 68, 120
    H, W = 16 * h, 16 * w
    res = []

    def rec(name, ms, bytes_moved):
        res.append(dict(kernel=name, ms=round(ms, 4), GBps=round(bytes_moved / ms / 1e6, 1), MB=round(bytes_moved / 1e6, 1)))

    # the decoder's residual stream is a fp16 (hi, lo) pair: 4 bytes per element read, raw + raw_lo + relu written
    def pair(*shape):
        return torch.randn(*shape, device=dev).half(), (torch.randn(*shape, device=dev) * 1e-3).half()
    p16, p16_lo = pair(K, h, w, 512); skip8, skip8_lo = pair(1, 2 * h, 2 * w, 512)
    rec('up2_add_split 1/16->1/8 (512ch)', timeit(lambda: ops.up2_add_split(p16, p16_lo, skip8, skip8_lo)),
        p16.numel() * 4 + skip8.numel() * 4 + 3 * K * 4 * h * w * 512 * 2)
    p8, p8_lo = pair(K, 2 * h, 2 * w, 256); skip4, skip4_lo = pair(1, 4 * h, 4 * w, 256)
    rec('up2_add_split 1/8->1/4 (256ch, + e4m3 relu remainder)',
        timeit(lambda: ops.up2_add_split(p8, p8_lo, skip4, skip4_lo, want_relu_lo8=True)),
        p8.numel() * 4 + skip4.numel() * 4 + 7 * K * 16 * h * w * 256)
    p4 = torch.randn(K, 4 * h, 4 * w, 256, device=dev).half()
    rec('area_down x4 (256ch @1/4)', timeit(lambda: ops.area_down(p4, 4)), p4.numel() * 2 * (1 + 1 / 16))
    rec('area_down x2 (256ch @1/8)', timeit(lambda: ops.area_down(p8, 2)), p8.numel() * 2 * 1.25)
    img = torch.randn(1, 3, H, W, device=dev)
    rec('stem_im2col image (hi+lo, K=192)', timeit(lambda: ops.stem_columns(img, 192, with_lo=True)), img.numel() * 4 + 2 * (H // 2) * (W // 2) * 192 * 2)
    masks = torch.rand(K, 1, H, W, device=dev)
    rec('stem_im2col masks (K=64)', timeit(lambda: ops.stem_columns(masks, 64)), masks.numel() * 4 + K * (H // 2) * (W // 2) * 64 * 2)
    x2 = torch.randn(K, H // 2, W // 2, 64, device=dev).half()
    rec('maxpool 3x3s2 (64ch @1/2)', timeit(lambda: ops.maxpool(x2)), x2.numel() * 2 * 1.25)
    cb = dict(w1=torch.randn(32, 512, device=dev), b1=torch.randn(32, device=dev), w2=torch.randn(512, 32, device=dev),
              b2=torch.randn(512, device=dev), ws=torch.randn(98, device=dev), bs=torch.randn(1, device=dev))
    # (hi, lo) read by the pooling, the statistics and the apply pass; raw + raw_lo + relu written
    rec('cbam_residual_split (512ch @1/16)', timeit(lambda: ops.cbam_residual_split(p16, p16_lo, cb)), p16.numel() * 2 * 9)
    logits = torch.randn(K, 4 * h, 4 * w, device=dev); agg = torch.empty(K + 1, 4 * h, 4 * w, device=dev)
    prob = torch.empty(K + 1, H, W, device=dev)
    rec('aggregate + x4 + softmax', timeit(lambda: nat.output_tail(logits, agg, prob, None, K, 4 * h, 4 * w)), logits.numel() * 4 * 2 + agg.numel() * 4 + prob.numel() * 4)
    n = h * w
    key = torch.randn(64, n, device=dev); shr = torch.rand(n, device=dev) + 1
    k_hi = torch.empty(n, 128, dtype=torch.float16, device=dev); k_lo = torch.empty_like(k_hi)
    ns = torch.empty(n, device=dev); rk = torch.empty(n, 64, device=dev); rs = torch.empty(n, device=dev); rsel = torch.empty(n, 64, device=dev)
    rec('pack_keys (bank append, 1 frame)', timeit(lambda: nat.pack_keys(key, key, n, 1, shr, 64, n, k_hi, k_lo, ns, rk, rsel, rs)), n * (64 * 4 * 2 + 4 + 128 * 2 * 2 + 4 + 64 * 4 * 2 + 4))
    v = torch.randn(n, 512, device=dev).half(); bank = torch.zeros(512, 100000, dtype=torch.float16, device=dev)
    rec('transpose_append (value append, 1 object)', timeit(lambda: nat.transpose_append(v, bank[:, 8000:], 100000, n, 512)), n * 512 * 2 * 2)
    for r in res:
        print(json.dumps(r))


if __name__ == '__main__':
    main()
