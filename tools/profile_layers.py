"""Per-layer CUDA-event timing of one propagated frame at a BASELINE config (native conv stack).

    python tools/profile_layers.py [--workload c3] [--frames 6]
Prints a table: layer / op, calls per frame, ms per frame, achieved TFLOP/s (convs) and share of the frame.
"""
import argparse, collections, json, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tracking-anything-with-deva_b200'))
import bench  # noqa: E402
from deva import _native as nat  # noqa: E402
from deva.model import native_ops as ops  # noqa: E402

records = []


def timed(name, flops, fn, *a, **kw):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); out = fn(*a, **kw); e1.record()
    records.append((name, flops, e0, e1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='c3')
    ap.add_argument('--frames', type=int, default=5)
    a = ap.parse_args()
    wl = bench.WORKLOADS[a.workload]
    dev = torch.device('cuda', 0)
    clip = bench.Clip(wl, dev, seed=100)
    eng = clip.core.network.engine
    names = {id(pc): n for n, pc in eng.P.items()}
    orig_conv = ops.conv_ex

    def conv_ex(x, pc, **kw):
        b, h, w, _ = x.shape
        ho, wo = pc.out_hw(h, w)
        passes = 3 if pc.precise else (2 if (pc.two_inputs or pc.w_lo) else 1)
        fl = 2.0 * b * ho * wo * pc.cout * pc.k * pc.k * pc.cin_pad * passes  # EXECUTED flops (all MMA passes)
        if kw.get('ksplit', 0) > 1:  # inner call of a chained split-precision conv: already inside the outer record
            return orig_conv(x, pc, **kw)
        return timed('conv:' + names.get(id(pc), '?') + (f' [{passes} passes]' if passes > 1 else ''), fl, orig_conv, x, pc, **kw)
    ops.conv_ex = conv_ex
    for fn in ('maxpool', 'up2_add_split', 'area_down', 'area_down_plane', 'cbam_residual_split', 'stem_columns'):
        o = getattr(ops, fn)
        setattr(ops, fn, (lambda o, fn: lambda *aa, **kw: timed('ew:' + fn, 0, o, *aa, **kw))(o, fn))
    for fn in ('pack_query', 'sim_topk', 'readout', 'output_tail', 'key_tail', 'pack_keys', 'transpose_append', 'nchw_to_nhwc', 'readout_sparse', 'head_gather3x3'):
        o = getattr(nat, fn)
        setattr(nat, fn, (lambda o, fn: lambda *aa, **kw: timed('mem:' + fn if fn in ('pack_query', 'sim_topk', 'readout', 'readout_sparse', 'pack_keys', 'transpose_append') else 'ew:' + fn, 0, o, *aa, **kw))(o, fn))
    for _ in range(6):  # one full mem_every period: the first regular memory frame (allocator growth) stays out of the table
        clip.step_resident()
    torch.cuda.synchronize()
    records.clear()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.frames):
        clip.step_resident()
    e1.record()
    torch.cuda.synchronize()
    total = e0.elapsed_time(e1) / a.frames
    agg = collections.OrderedDict()
    for name, fl, s, e in records:
        r = agg.setdefault(name, [0, 0.0, 0.0])
        r[0] += 1; r[1] += s.elapsed_time(e); r[2] += fl
    rows = sorted(agg.items(), key=lambda kv: -kv[1][1])
    kern = sum(v[1] for v in agg.values()) / a.frames
    print(f'# {wl["name"]}: {total:.2f} ms/frame wall (events), {kern:.2f} ms in timed ops, {a.frames} frames (1 in 5 is a memory frame)')
    print(f'{"op":58s} {"calls/f":>8s} {"ms/frame":>9s} {"TFLOP/s":>8s} {"share":>6s}')
    for name, (c, ms, fl) in rows[:45]:
        tf = fl / (ms * 1e-3) / 1e12 if fl else 0
        print(f'{name:58s} {c / a.frames:8.1f} {ms / a.frames:9.3f} {tf:8.0f} {100 * ms / a.frames / total:5.1f}%')
    convs = [(n, v) for n, v in agg.items() if n.startswith('conv:')]
    cms = sum(v[1] for _, v in convs); cfl = sum(v[2] for _, v in convs)
    print(f'# all convs: {cms / a.frames:.2f} ms/frame, {cfl / (cms * 1e-3) / 1e12:.0f} TFLOP/s aggregate; '
          f'memory read+bank: {sum(v[1] for n, v in agg.items() if n.startswith("mem:")) / a.frames:.2f} ms; '
          f'helpers: {sum(v[1] for n, v in agg.items() if n.startswith("ew:")) / a.frames:.2f} ms')


if __name__ == '__main__':
    main()
