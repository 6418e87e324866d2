"""VIPSeg evaluation after inference - stuff merging, VPQ at seven window sizes, STQ - the reference's and this package's.

    python tools/bench_vps_metrics.py [--videos 4] [--frames 25] [--segments 60]

Input: a seeded synthetic dataset shaped like VIPSeg (tests/golden/vps_scenario.py's generator at 720x1280, --videos
videos of --frames frames, about --segments listed segments per frame: some of the drawn things end up occluded), written to a temporary directory that is removed
afterwards.

Reference: the unmodified modules staged under oracle/_ref (oracle/build_ref_vps.py), loaded by path as tools/bench_saver.py
does: ``process_single_video`` serially per video (its ``merge_stuff`` maps the same function over Pool(16)),
``eval_vpq`` with ``num_processes`` = min(16, CPUs) and ``eval_stq`` (single process).  Ours: ``merge_stuff``,
``eval_vpq``, ``eval_stq`` and ``eval_vps`` (both metrics from one decode pass), then the parts of one pass measured
separately: PNG decode on the thread pool, upload through pinned buffers, the joint-histogram kernels (CUDA events, with
the frames resident) and the host matching.  Prints one JSON line with the card and its power limit read in the same
run.  The kernels' rate counts the bytes they must read: two RGB frames per frame pair."""
import argparse
import importlib.util
import json
import os
import shutil
import sys
import tempfile
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, 'oracle', '_ref')
sys.path.insert(0, ROOT)
import bench  # noqa: E402,F401  (puts the package on sys.path)
sys.path.append(REF)  # after the package: only what the package lacks resolves there
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import vps_scenario as vs  # noqa: E402
from bench_ingest import card  # noqa: E402

HBM_TBS = 3.35


def load_reference():
    mods = {}
    for name in ('eval_vpq_vipseg', 'eval_stq_vipseg', 'stuff_merging'):
        path = os.path.join(REF, 'deva', 'vps_metrics', name + '.py')
        if not os.path.isfile(path):
            raise RuntimeError('oracle/_ref/deva/vps_metrics is not staged: run python oracle/build_ref.py and '
                               'oracle/build_ref_vps.py in the build container')
        spec = importlib.util.spec_from_file_location('ref_' + name, path)  # not deva.*: that name is this package's
        mods[name] = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = mods[name]  # eval_vpq's Pool pickles its worker function by module name
        spec.loader.exec_module(mods[name])
    return mods


def make_dataset(root, videos, frames, segments):
    vs.VIDEOS = {f'b{i}': (frames, 720, 1280, segments + 15, 100 + i) for i in range(videos)}
    return vs.write_dataset(root)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def parts(submit, truth, gt_path):
    """One pass split into decode, upload, kernels and host matching."""
    from deva import _native as nat
    from deva.vps_metrics import scoring, video_pass
    _, videos = video_pass.load_dataset(submit, truth, gt_path)
    categories = {el['id']: el for el in json.load(open(gt_path))['categories']}
    things = scoring.thing_list(json.load(open(gt_path))['categories'])
    dec = video_pass.Decoder()
    t0 = time.perf_counter()
    decoded = [(list(dec.frames(g)), list(dec.frames(p))) for _, _, _, g, p in videos]
    decode_s = time.perf_counter() - t0
    dec.close()
    upload = video_pass.Uploader(torch.device('cuda'))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    on_dev = [([upload(a) for a in g], [upload(a) for a in p]) for g, p in decoded]
    torch.cuda.synchronize()
    upload_s = time.perf_counter() - t0
    tables = [(torch.from_numpy(scoring.id_table(gj)).cuda(), torch.from_numpy(scoring.id_table(pj)).cuda())
              for _, gj, pj, _, _ in videos]
    hists = [torch.empty(len(g), len(gi) + 1, len(pi) + 1, dtype=torch.int32, device='cuda')
             for (g, _), (gi, pi) in zip(on_dev, tables)]

    def kernels():
        for (g, p), (gi, pi), h in zip(on_dev, tables, hists):
            for t in range(len(g)):
                nat.pano_joint_hist(g[t], p[t], gi, pi, h[t])

    kernels()
    reps = 5
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        kernels()
    e1.record()
    torch.cuda.synchronize()
    kernel_s = e0.elapsed_time(e1) / 1e3 / reps
    host = [h.cpu().numpy() for h in hists]
    t0 = time.perf_counter()
    stq = scoring.STQuality(things)
    for seq, ((vid, gj, pj, _, pp), (gi, pi), h) in enumerate(zip(videos, tables, host)):
        gi, pi = gi.cpu().numpy(), pi.cpu().numpy()
        video = scoring.VpqVideo(gj, pj, gi, pi, h, categories, video_pass.png_labels(pp))
        for n in scoring.NFRAMES:
            video.stat(n)
        stq.update_video(seq, gj, pj, gi, pi, h)
    stq.result()
    host_s = time.perf_counter() - t0
    n_frames = sum(len(g) for g, _ in decoded)
    px = sum(a.size for g, p in decoded for a in g + p)
    return {'decode_ms': round(decode_s * 1e3, 1), 'upload_ms': round(upload_s * 1e3, 1),
            'kernels_ms': round(kernel_s * 1e3, 3), 'host_matching_ms': round(host_s * 1e3, 1),
            'kernel_tb_s': round(px / kernel_s / 1e12, 3), 'kernel_share_of_3.35tb_s': round(px / kernel_s / 1e12 / HBM_TBS, 3),
            'frames': n_frames, 'decode_threads': dec.pool._max_workers}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--videos', type=int, default=4)
    ap.add_argument('--frames', type=int, default=25)
    ap.add_argument('--segments', type=int, default=60)
    args = ap.parse_args()
    from deva import _native as nat
    nat.require_device()
    ref = load_reference()
    from deva.vps_metrics import eval_vps
    from deva.vps_metrics.eval_stq_vipseg import eval_stq
    from deva.vps_metrics.eval_vpq_vipseg import eval_vpq
    from deva.vps_metrics.stuff_merging import merge_stuff
    n_proc = min(16, os.cpu_count() or 1)
    root = tempfile.mkdtemp()
    try:
        submit, truth, gt_path = make_dataset(root, args.videos, args.frames, args.segments)
        isthing = dict(vs.ISTHING)
        ref['stuff_merging'].vipseg_cat_to_isthing = isthing
        anns = json.load(open(os.path.join(submit, 'pred.json')))['annotations']
        out = {}
        t = {}
        ref_merged = []
        np.random.seed(0)
        t['ref_merge'] = timed(lambda: ref_merged.extend(ref['stuff_merging'].process_single_video(a, submit,
                                                                                                   root + '/m_ref')
                                                         for a in anns))
        np.random.seed(0)
        t['ours_merge'] = timed(lambda: merge_stuff(submit, root + '/m_ours', isthing=isthing))
        t['ours_vpq'] = timed(lambda: eval_vpq(submit, truth, gt_path))
        t['ours_stq'] = timed(lambda: eval_stq(submit, truth, gt_path))
        ours_files = {n: open(os.path.join(submit, n)).read() for n in os.listdir(submit) if n.endswith('.txt')}
        t['ours_vps'] = timed(lambda: eval_vps(submit, truth, gt_path))
        t['ref_vpq'] = timed(lambda: ref['eval_vpq_vipseg'].eval_vpq(submit, truth, gt_path, num_processes=n_proc))
        t['ref_stq'] = timed(lambda: ref['eval_stq_vipseg'].eval_stq(submit, truth, gt_path))
        ref_files = {n: open(os.path.join(submit, n)).read() for n in os.listdir(submit) if n.endswith('.txt')}
        out['merge_json_equal'] = json.load(open(root + '/m_ours/pred.json')) == {'annotations': ref_merged}
        out['card'] = card()
        out['cpu_threads'] = os.cpu_count()
        out['dataset'] = {'videos': args.videos, 'frames': args.frames, 'size': [720, 1280],
                          'segments_per_frame': args.segments}
        out['per_video_s'] = {k: round(v / args.videos, 3) for k, v in t.items()}
        out['files_equal'] = ours_files == ref_files
        out['ours_pass_parts_per_video_ms'] = {k: (round(v / args.videos, 2) if k.endswith('_ms') else v)
                                               for k, v in parts(submit, truth, gt_path).items()}
        print(json.dumps(out))
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == '__main__':
    main()
