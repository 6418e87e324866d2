"""STQ of VIPSeg (the reference's deva/vps_metrics/eval_stq_vipseg.py) from one joint label histogram per frame.
Writes stq.txt byte for byte as the reference does.

evaluation/eval_with_detections.py runs eval_stq in a multiprocessing.Process forked after CUDA has been initialised,
and CUDA cannot start in such a child.  There eval_stq runs its device pass in a freshly spawned process, with the same
png_decoder, and waits."""
import multiprocessing
import os

import torch

from deva.utils.png_decode import resolve_decoder
from deva.vps_metrics import video_pass


def eval_stq(submit_dir, truth_dir, pan_gt_json_file, *, png_decoder=None):
    """png_decoder: 'pil' or 'device'; None reads DEVA_B200_PNG_DECODER (default 'pil')."""
    png_decoder = resolve_decoder(png_decoder)
    if torch.cuda._is_in_bad_fork():
        child = multiprocessing.get_context('spawn').Process(target=eval_stq,
                                                             args=(submit_dir, truth_dir, pan_gt_json_file),
                                                             kwargs={'png_decoder': png_decoder})
        child.start()
        child.join()
        if child.exitcode != 0:
            raise RuntimeError(f'eval_stq: the spawned evaluation exited with code {child.exitcode}')
        return
    if not os.path.isdir(submit_dir):
        print("%s doesn't exist" % submit_dir)
    _, stq_metric, _ = video_pass.evaluate(submit_dir, truth_dir, pan_gt_json_file, vpq=False, png_decoder=png_decoder)
    video_pass.write_stq(submit_dir, stq_metric)
