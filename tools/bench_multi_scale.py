"""Per-frame cost of multi-scale / flip evaluation on 1080p frames: the six-member ensemble {480, 600, 720} x flip.

    python tools/bench_multi_scale.py [--steps 20] [--warmup 5] [--reps 50]

  * ensemble: MultiScaleCore over pinned 1080p uint8 frames with 5 objects (first frame with its mask, then plain
    steps), the merged uint8 id map copied to the host every frame; wall time per frame.
  * egress:   the kernels alone from CUDA events - six prob_to_scores calls (each member's [6, h, w] probabilities
    resized back to 1080x1920, flipped back for the flipped members, added into one int32 sum) and one scores_to_ids
    - with their DRAM bytes (probabilities read once, the sum read and written per member, read once by the merge,
    the ids written) against the H100 SXM's 3.35 TB/s.
  * reference: the reference's export and merge for the same six arrays: device F.interpolate + flip,
    ``(prob.cpu().numpy() * 255).astype(np.uint8)`` per member (eval_vos.py:169-189, files not written), then
    merge_multi_scale.py's float32 sum, np.argmax and remap loop; wall time per frame.
Prints one JSON line with the card and its power limit read in the same run."""
import argparse
import json
import os
import sys
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import bench  # noqa: E402  (puts the package on sys.path)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from bench_ingest import card, event_ms  # noqa: E402

H0, W0, K = 1080, 1920, 5
MEMBERS = [(size, flip) for size in (480, 600, 720) for flip in (False, True)]
PEAK_BPS = 3.35e12


def frames_and_mask(n):
    g = torch.Generator().manual_seed(0)
    frames = [torch.randint(0, 256, (H0, W0, 3), generator=g, dtype=torch.uint8).pin_memory() for _ in range(n)]
    mask = torch.zeros(H0, W0, dtype=torch.uint8)
    for k in range(K):
        mask[100 + 150 * k: 250 + 150 * k, 200 + 300 * k: 500 + 300 * k] = k + 1
    return frames, mask.pin_memory()


def ensemble(steps, warmup):
    from deva.inference.frame_io import reader_size
    from deva.inference.multi_scale import MultiScaleCore
    net = bench.make_network(torch.device('cuda', 0))
    ms = MultiScaleCore(net, bench.base_config(), MEMBERS)
    frames, mask = frames_and_mask(5)
    ms.step(frames[0], mask, list(range(1, K + 1))).cpu()
    for i in range(warmup):
        ms.step(frames[(i + 1) % 5]).cpu()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        ms.step(frames[(i + 1) % 5]).cpu()
    torch.cuda.synchronize()
    ms_frame = (time.perf_counter() - t0) * 1e3 / steps
    shapes = [reader_size(H0, W0, size) for size, _ in MEMBERS]
    return {'ms_per_frame': round(ms_frame, 2), 'fps': round(1e3 / ms_frame, 3), 'member_shapes': shapes,
            'mapping': ms.object_manager.get_tmp_to_obj_mapping()}


def member_probs(shapes):
    g = torch.Generator(device='cuda').manual_seed(1)
    out = []
    for h, w in shapes:
        p = torch.softmax(4 * torch.randn(K + 1, h // 16, w // 16, device='cuda', generator=g), 0)
        out.append(F.interpolate(p[None], (h, w), mode='bilinear', align_corners=False)[0].contiguous())
    return out


def egress(probs, mapping, reps):
    from deva.inference.frame_io import prob_to_scores, scores_to_ids
    total = torch.zeros(K + 1, H0, W0, dtype=torch.int32, device='cuda')

    def export():
        for p, (_, flip) in zip(probs, MEMBERS):
            prob_to_scores(p, (H0, W0), flip, scores=False, into=total)

    def merge():
        scores_to_ids(total, mapping=mapping)

    export_ms, merge_ms = event_ms(export, reps), event_ms(merge, reps)
    plane = (K + 1) * H0 * W0
    export_bytes = sum(p.numel() * 4 for p in probs) + len(probs) * 2 * plane * 4
    merge_bytes = plane * 4 + H0 * W0
    return {'export_6_members_ms': round(export_ms, 4), 'merge_ms': round(merge_ms, 4),
            'export_GBps': round(export_bytes / export_ms / 1e6, 1), 'merge_GBps': round(merge_bytes / merge_ms / 1e6, 1),
            'export_frac_of_peak': round(export_bytes / export_ms * 1e3 / PEAK_BPS, 3),
            'merge_frac_of_peak': round(merge_bytes / merge_ms * 1e3 / PEAK_BPS, 3)}


def reference_export(probs, mapping, n):
    def one():
        total = None
        for p, (_, flip) in zip(probs, MEMBERS):
            prob = F.interpolate(p.unsqueeze(1), (H0, W0), mode='bilinear', align_corners=False)[:, 0]
            if flip:
                prob = torch.flip(prob, dims=[-1])
            s = (prob.detach().cpu().numpy() * 255).astype(np.uint8)
            total = s.astype(np.float32) if total is None else total + s
        result = np.argmax(total, axis=0)
        idx = np.zeros_like(result, dtype=np.uint8)
        for l, i in mapping.items():
            idx[result == i] = l
        return idx

    one()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        one()
    return round((time.perf_counter() - t0) * 1e3 / n, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--reps', type=int, default=50)
    args = ap.parse_args()
    from deva import _native as nat
    nat.require_device()
    torch.set_grad_enabled(False)
    run = ensemble(args.steps, args.warmup)
    probs = member_probs(run['member_shapes'])
    out = {'card': card(), 'members': MEMBERS, 'objects': K, 'input': f'{W0}x{H0} uint8',
           'ensemble': run, 'egress_kernels': egress(probs, run['mapping'], args.reps),
           'reference_export_and_merge_ms_per_frame': reference_export(probs, run['mapping'], 5)}
    out['ensemble']['mapping'] = {str(k): v for k, v in run['mapping'].items()}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
