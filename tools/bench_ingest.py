"""Per-frame cost of getting a decoded frame to the working resolution on the device, and one end-to-end 480p loop.

    python tools/bench_ingest.py [--frames 60] [--e2e-steps 100]

For 1080p and 4K uint8 host frames resized to a short side of 480:
  * host:   the reference readers' path - torchvision ToTensor + Normalize + Resize(480, BILINEAR, antialias=True) on
            the CPU (1 thread, as in one DataLoader worker, and all threads) plus the H2D copy of the float frame;
  * torch:  pinned uint8 H2D, normalise and F.interpolate(antialias=True) with torch on the GPU;
  * ours:   pinned uint8 H2D + frame_from_rgb8(size=480), and the kernels alone from CUDA events.
End to end: 1080p uint8 host frames -> frame_from_rgb8(size=480) -> step (bench.py's c2 setup: 5 objects, 2k slots,
at the 480x853 the ingest produces) -> prob_to_ids(size=1080x1920) -> D2H.  Prints one JSON line with the card and its
power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (puts the package on sys.path)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=name,power.limit,clocks.max.sm',
                               '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f'unavailable ({e})'


def host_ms(fn, n):
    fn()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def event_ms(fn, n):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def ingest_rows(n, size=480):
    from PIL import Image
    from torchvision import transforms
    from deva.inference.frame_io import IMAGENET_MEAN, IMAGENET_STD, frame_from_rgb8
    reader = transforms.Compose([transforms.ToTensor(), transforms.Normalize(IMAGENET_MEAN, IMAGENET_STD),
                                 transforms.Resize(size, interpolation=transforms.InterpolationMode.BILINEAR,
                                                   antialias=True)])
    mean = torch.tensor(IMAGENET_MEAN, device='cuda').view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD, device='cuda').view(1, 3, 1, 1)
    rows = {}
    threads = torch.get_num_threads()
    for name, (h, w) in (('1080p', (1080, 1920)), ('4k', (2160, 3840))):
        g = torch.Generator().manual_seed(0)
        frame = torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8)
        pil = Image.fromarray(frame.numpy())
        pinned = frame.pin_memory()
        on_dev = pinned.cuda()
        out_shape = tuple(frame_from_rgb8(on_dev, size=size).shape)
        row = {'out': out_shape}
        for label, nt in (('host_1thread_ms', 1), ('host_all_threads_ms', threads)):
            torch.set_num_threads(nt)
            row[label] = host_ms(lambda: reader(pil), max(3, n // 4))
        torch.set_num_threads(threads)
        host_float = reader(pil)
        row['h2d_float_ms'] = host_ms(lambda: host_float.cuda(), n)

        def torch_gpu():
            x = pinned.cuda(non_blocking=True).permute(2, 0, 1)[None].float().div(255)
            return F.interpolate((x - mean) / std, out_shape[1:], mode='bilinear', align_corners=False, antialias=True)
        row['torch_gpu_ms'] = host_ms(torch_gpu, n)
        row['ours_ms'] = host_ms(lambda: frame_from_rgb8(pinned, size=size), n)
        row['ours_kernel_ms'] = event_ms(lambda: frame_from_rgb8(on_dev, size=size), 10 * n)
        row['h2d_u8_pinned_ms'] = event_ms(lambda: pinned.cuda(non_blocking=True), n)
        rows[name] = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in row.items()}
    return rows


def e2e(steps, warmup):
    from deva.inference.frame_io import frame_from_rgb8, prob_to_ids
    wl = dict(bench.WORKLOADS['c2'], w=853)  # frame_from_rgb8(size=480)'s output for a 1920x1080 frame
    clip = bench.Clip(wl, torch.device('cuda', 0), seed=0)
    g = torch.Generator().manual_seed(1)
    frames = [torch.randint(0, 256, (1080, 1920, 3), generator=g, dtype=torch.uint8).pin_memory() for _ in range(5)]

    def one(i):
        img = frame_from_rgb8(frames[i % 5], size=480)
        p = clip.core.step(img)
        ids = prob_to_ids(p, clip.core.object_manager, size=(1080, 1920), dtype=torch.uint8).cpu()
        clip.clamp()
        return ids

    for i in range(warmup):
        one(i)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        one(i)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    return {'workload': 'c2-like: 1080p uint8 in, 480x853 working size, 5 objects, 2k slots, 1080p id map out',
            'ms_per_frame': round(ms, 3), 'fps': round(1e3 / ms, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=60)
    ap.add_argument('--e2e-steps', type=int, default=100)
    ap.add_argument('--e2e-warmup', type=int, default=10)
    args = ap.parse_args()
    from deva import _native as nat
    nat.require_device()
    torch.set_grad_enabled(False)
    out = {'card': card(), 'cpu_threads': torch.get_num_threads(), 'ingest': ingest_rows(args.frames),
           'e2e_480p': e2e(args.e2e_steps, args.e2e_warmup)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
