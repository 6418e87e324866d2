"""Where the key path of a propagated frame goes: encode_image + transform_key at a BASELINE config.

    python tools/profile_key_path.py [--workload c3] [--frames 10] [--out DIR]

Reports, per frame of the workload:
  - the key path's wall time (CUDA events around the two calls, inside the frame as bench.py runs it) and the frame's;
  - the sum of the key path's kernel times (torch.profiler, in a run of its own);
  - one row per conv2d launch: layer, pixel tiles x channel tiles x k-splits = work units against the SM count, the
    pixel tile (th, tw) and its time (CUDA events around the single launch, a third run).
"""
import argparse, collections, json, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tracking-anything-with-deva_b200'))
import bench  # noqa: E402
from deva import _native as nat  # noqa: E402
from deva.model import native_ops as ops  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='c3')
    ap.add_argument('--frames', type=int, default=10)
    ap.add_argument('--out', default=None, help='directory for the JSON summary')
    a = ap.parse_args()
    wl = bench.WORKLOADS[a.workload]
    dev = torch.device('cuda', 0)
    clip = bench.Clip(wl, dev, seed=100)
    eng = clip.core.network.engine
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    names = {id(pc): n for n, pc in eng.P.items()}

    # 1. wall time of the key path inside the frame: events around encode_image and transform_key
    spans, mode = [], {'on': False}
    orig = {fn: getattr(eng, fn) for fn in ('encode_image', 'transform_key')}

    def wrap(fn):
        def f(*aa, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); out = orig[fn](*aa, **kw); e1.record()
            if mode['on']:
                spans.append((fn, e0, e1))
            return out
        return f
    for fn in orig:
        setattr(eng, fn, wrap(fn))
    for _ in range(6):  # one full mem_every period of warm-up
        clip.step_resident()
    torch.cuda.synchronize()
    mode['on'] = True
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    f0.record()
    for _ in range(a.frames):
        clip.step_resident()
    f1.record()
    torch.cuda.synchronize()
    mode['on'] = False
    frame_ms = f0.elapsed_time(f1) / a.frames
    per_fn = collections.Counter()
    for fn, e0, e1 in spans:
        per_fn[fn] += e0.elapsed_time(e1) / a.frames
    calls = collections.Counter(fn for fn, _, _ in spans)
    wall = per_fn['encode_image'] + per_fn['transform_key']

    # 2. kernel time of the key path alone (same frame, same shapes), under the profiler
    img = clip.frames_dev[0:1]

    def key_path():
        _, feat = eng.encode_image(img)
        eng.transform_key(feat)
    for _ in range(3):
        key_path()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    reps = 5
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            key_path()
        torch.cuda.synchronize()
    kern = collections.Counter()
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            kern[ev.name] += ev.device_time / 1e3 / reps  # us -> ms
    kern_ms = sum(kern.values())

    # 3. per conv2d launch: units against the SMs, and its time alone
    cur = {'name': '?'}
    orig_conv_ex, orig_conv2d = ops.conv_ex, nat.conv2d
    launches = []

    def conv_ex(x, pc, **kw):
        outer, cur['name'] = cur['name'], names.get(id(pc), '?')
        try:
            return orig_conv_ex(x, pc, **kw)
        finally:
            cur['name'] = outer

    def conv2d(x, batch, h, w, cin_pad, w_packed, kh, stride, cout, cout_pad, nt, th, tw, *aa, **kw):
        ho, wo = (h + 2 * (kh // 2) - kh) // stride + 1, (w + 2 * (kh // 2) - kh) // stride + 1
        tiles = batch * ops.pixel_tiles(ho, wo, (th, tw))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        orig_conv2d(x, batch, h, w, cin_pad, w_packed, kh, stride, cout, cout_pad, nt, th, tw, *aa, **kw)
        e1.record()
        launches.append(dict(layer=cur['name'], pixel_tiles=tiles, tile=[th, tw], nt=nt, channel_tiles=cout_pad // nt,
                             ksplit=max(kw.get('ksplit', 0), 1), ev=(e0, e1)))
    ops.conv_ex, nat.conv2d = conv_ex, conv2d
    try:
        key_path(); torch.cuda.synchronize(); launches.clear()
        for _ in range(reps):
            key_path()
        torch.cuda.synchronize()
    finally:
        ops.conv_ex, nat.conv2d = orig_conv_ex, orig_conv2d
    n = len(launches) // reps
    rows = []
    for i in range(n):
        r = dict(launches[i]); r.pop('ev')
        r['units'] = r['pixel_tiles'] * r['channel_tiles'] * r['ksplit']
        r['ms'] = sum(launches[i + j * n]['ev'][0].elapsed_time(launches[i + j * n]['ev'][1]) for j in range(reps)) / reps
        rows.append(r)

    props = torch.cuda.get_device_properties(dev)
    print(f'# {wl["name"]}: {props.name}, {sms} SMs')
    print(f'# frame {frame_ms:.2f} ms; key path wall {wall:.3f} ms/frame ({100 * wall / frame_ms:.1f} %): '
          f'encode_image {per_fn["encode_image"]:.3f} ms x {calls["encode_image"] / a.frames:.1f}, '
          f'transform_key {per_fn["transform_key"]:.3f} ms x {calls["transform_key"] / a.frames:.1f}')
    print(f'# key path kernel time {kern_ms:.3f} ms per call ({len(rows)} conv launches, sum of their times '
          f'{sum(r["ms"] for r in rows):.3f} ms when timed one by one)')
    print(f'{"layer":44s} {"tile":>8s} {"px x ch x ks":>14s} {"units":>6s} {"waves":>6s} {"ms":>7s}')
    for r in rows:
        print(f'{r["layer"]:44s} {str(tuple(r["tile"])):>8s} '
              f'{r["pixel_tiles"]:>4d}x{r["channel_tiles"]}x{r["ksplit"]:<4d} {r["units"]:6d} {r["units"] / sms:6.2f} {r["ms"]:7.3f}')
    top = sorted(kern.items(), key=lambda kv: -kv[1])[:12]
    print('# kernels by time (ms per call):', ', '.join(f'{k[:40]} {v:.3f}' for k, v in top))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, f'key_path_{a.workload}.json'), 'w') as f:
            json.dump(dict(gpu=props.name, sms=sms, frame_ms=frame_ms, key_wall_ms=wall, per_fn=dict(per_fn),
                           key_kernel_ms=kern_ms, launches=rows), f, indent=1)


if __name__ == '__main__':
    main()
