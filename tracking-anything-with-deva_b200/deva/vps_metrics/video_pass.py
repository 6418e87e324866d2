"""The one per-video device pass behind VPQ, STQ and stuff merging.

PNGs are decoded with PIL on a pool of host threads (in order, ahead of use), copied into a ring of pinned staging
buffers and uploaded, or with ``png_decoder='device'`` (``DEVA_B200_PNG_DECODER=device``) decoded a video at a time on
the device (png_pipeline.DeviceDecoder); each frame pair is reduced by ``deva_b200_pano_joint_hist`` into its slice of one int32
``[T, G + 1, P + 1]`` buffer, and that buffer comes to the host once per video.  Importing this module does not
initialise CUDA.
"""
import json
import os

import numpy as np
import torch
from PIL import Image

from deva.utils import png_pipeline
from deva.utils.png_decode import resolve_decoder
from deva.utils.png_pipeline import RING, Uploader  # noqa: F401  (part of this module's interface)
from deva.vps_metrics import scoring


def read_rgb(path) -> np.ndarray:
    """uint8 [h, w, 3] of an RGB id PNG (np.array(Image.open(path)) as the reference reads it)."""
    a = np.asarray(Image.open(path))
    if a.ndim != 3 or a.shape[2] < 3:
        raise ValueError(f'{path}: expected an RGB id image, got shape {a.shape}')
    return np.ascontiguousarray(a[:, :, :3])


class Decoder(png_pipeline.Decoder):
    """The thread pool decoding RGB id PNGs (read_rgb)."""

    def __init__(self, num_threads=None):
        super().__init__(read_rgb, num_threads)


def make_decoder(png_decoder, device, num_threads=None):
    """The frame source of RGB id PNGs: Decoder for 'pil', the device's for 'device' (RGB and RGBA files; every other
    file goes through read_rgb and raises its error)."""
    if png_decoder == 'device':
        return png_pipeline.DeviceDecoder(read_rgb, device, modes=('RGB', 'RGBA'), rgb=True, num_threads=num_threads)
    return Decoder(num_threads)


def require_device():
    from deva import _native
    _native.require_device()
    return torch.device('cuda', torch.cuda.current_device())


def video_histograms(decoder, upload, gt_paths, pred_paths, gt_ids, pred_ids):
    """-> int32 [T, len(gt_ids) + 1, len(pred_ids) + 1]: the joint histogram of every frame pair, on the host."""
    from deva import _native
    dev = upload.device
    g = torch.from_numpy(gt_ids).to(dev, non_blocking=True)
    p = torch.from_numpy(pred_ids).to(dev, non_blocking=True)
    hist = torch.empty(len(gt_paths), len(gt_ids) + 1, len(pred_ids) + 1, dtype=torch.int32, device=dev)
    # one frame source over gt 0, pred 0, gt 1, ...: the order in which a pair's errors are met, and one batch of the
    # device decoder over both sides
    frames = decoder.frames([path for pair in zip(gt_paths, pred_paths) for path in pair])
    for t, (gt, pred) in enumerate(zip(frames, frames)):
        if tuple(gt.shape) != tuple(pred.shape):
            raise ValueError(f'{gt_paths[t]} and {pred_paths[t]} differ in size: {tuple(gt.shape)} vs '
                             f'{tuple(pred.shape)}')
        _native.pano_joint_hist(upload(gt), upload(pred), g, p, hist[t])
    return hist.cpu().numpy()


def load_dataset(submit_dir, truth_dir, pan_gt_json_file):
    """The reference evaluators' reading of the two JSON files: (categories list, [(video_id, gt frame entries, pred
    frame entries, gt paths, pred paths)]) in the GT file's video order."""
    with open(os.path.join(submit_dir, 'pred.json'), 'r') as f:
        pred_jsons = json.load(f)
    with open(pan_gt_json_file, 'r') as f:
        gt_jsons = json.load(f)
    pred_j = {a['video_id']: a['annotations'] for a in pred_jsons['annotations']}
    gt_j = {a['video_id']: a['annotations'] for a in gt_jsons['annotations']}
    videos = []
    for video in gt_jsons['videos']:
        vid = video['video_id']
        gt_js, pred_js = gt_j[vid], pred_j[vid]
        assert len(gt_js) == len(pred_js)
        names = [im['file_name'] for im in video['images']]
        videos.append((vid, gt_js, pred_js, [os.path.join(truth_dir, vid, n) for n in names],
                       [os.path.join(submit_dir, 'pan_pred', vid, n) for n in names]))
    return gt_jsons['categories'], videos


def png_labels(paths):
    """Error path of the prediction checks: the ascending ids of one prediction PNG, decoded on the host."""
    def labels(t):
        a = read_rgb(paths[t]).astype(np.uint32)
        return [int(v) for v in np.unique(a[:, :, 0] + a[:, :, 1] * 256 + a[:, :, 2] * 65536)]
    return labels


def evaluate(submit_dir, truth_dir, pan_gt_json_file, *, vpq=True, stq=True, num_threads=None, histograms=None,
             png_decoder=None):
    """One decode pass over the dataset.  -> ({nframes: PQStat} or None, STQuality or None, categories list).
    histograms(decoder, gt_paths, pred_paths, gt_ids, pred_ids) -> int [T, G + 1, P + 1]; default: the device pass.
    png_decoder: 'pil' or 'device'; None reads DEVA_B200_PNG_DECODER (default 'pil')."""
    png_decoder = resolve_decoder(png_decoder)
    categories_list, videos = load_dataset(submit_dir, truth_dir, pan_gt_json_file)
    categories = {el['id']: el for el in categories_list}
    dev = require_device() if histograms is None or png_decoder == 'device' else None
    if histograms is None:
        upload = Uploader(dev)

        def histograms(decoder, *args):
            return video_histograms(decoder, upload, *args)
    decoder = make_decoder(png_decoder, dev, num_threads)
    vpq_stats = {n: scoring.PQStat() for n in scoring.NFRAMES} if vpq else None
    stq_metric = scoring.STQuality(scoring.thing_list(categories_list)) if stq else None
    try:
        for seq_id, (vid, gt_js, pred_js, gt_paths, pred_paths) in enumerate(videos):
            gt_ids, pred_ids = scoring.id_table(gt_js), scoring.id_table(pred_js)
            hist = histograms(decoder, gt_paths, pred_paths, gt_ids, pred_ids)
            if vpq:
                video = scoring.VpqVideo(gt_js, pred_js, gt_ids, pred_ids, hist, categories, png_labels(pred_paths))
                for n in scoring.NFRAMES:
                    vpq_stats[n] += video.stat(n)
            if stq:
                stq_metric.update_video(seq_id, gt_js, pred_js, gt_ids, pred_ids, hist)
    finally:
        decoder.close()
    return vpq_stats, stq_metric, categories_list


def write_vpq(output_dir, vpq_stats, categories_list):
    categories = {el['id']: el for el in categories_list}
    vpqs = []
    for n in scoring.NFRAMES:
        results = scoring.vpq_results(vpq_stats[n], categories)
        with open(os.path.join(output_dir, 'vpq-%d.txt' % n), 'w') as f:
            f.write(scoring.vpq_text(results))
        vpqs.append((100 * results['All']['pq'], 100 * results['Things']['pq'], 100 * results['Stuff']['pq']))
        print('==> %d-frame vpq:' % n, *vpqs[-1])
    with open(os.path.join(output_dir, 'vpq-simple.txt'), 'w') as f:
        f.write(scoring.vpq_simple_text(vpqs))
    return vpqs


def write_stq(output_dir, stq_metric):
    result = stq_metric.result()
    print('STQ : {}'.format(result['STQ']))
    print('AQ :{}'.format(result['AQ']))
    print('IoU:{}'.format(result['IoU']))
    with open(os.path.join(output_dir, 'stq.txt'), 'w') as f:
        f.write(scoring.stq_text(result))
    return result


def eval_vps(submit_dir, truth_dir, pan_gt_json_file, num_processes=None, *, png_decoder=None):
    """VPQ at every window size and STQ from one decode pass: writes vpq-{n}.txt, vpq-simple.txt and stq.txt into
    submit_dir, as eval_vpq and eval_stq do.  num_processes: host decode threads.  png_decoder: 'pil' or 'device'; None
    reads DEVA_B200_PNG_DECODER (default 'pil')."""
    vpq_stats, stq_metric, categories_list = evaluate(submit_dir, truth_dir, pan_gt_json_file,
                                                      num_threads=num_processes, png_decoder=png_decoder)
    write_vpq(submit_dir, vpq_stats, categories_list)
    write_stq(submit_dir, stq_metric)
