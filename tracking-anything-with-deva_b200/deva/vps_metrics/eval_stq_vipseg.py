"""STQ of VIPSeg (the reference's deva/vps_metrics/eval_stq_vipseg.py) from one joint label histogram per frame.
Writes stq.txt byte for byte as the reference does.

evaluation/eval_with_detections.py runs eval_stq in a multiprocessing.Process forked after CUDA has been initialised,
and CUDA cannot start in such a child.  There eval_stq runs its device pass in a freshly spawned process and waits."""
import multiprocessing
import os

import torch

from deva.vps_metrics import video_pass


def eval_stq(submit_dir, truth_dir, pan_gt_json_file):
    if torch.cuda._is_in_bad_fork():
        child = multiprocessing.get_context('spawn').Process(target=eval_stq,
                                                             args=(submit_dir, truth_dir, pan_gt_json_file))
        child.start()
        child.join()
        if child.exitcode != 0:
            raise RuntimeError(f'eval_stq: the spawned evaluation exited with code {child.exitcode}')
        return
    if not os.path.isdir(submit_dir):
        print("%s doesn't exist" % submit_dir)
    _, stq_metric, _ = video_pass.evaluate(submit_dir, truth_dir, pan_gt_json_file, vpq=False)
    video_pass.write_stq(submit_dir, stq_metric)
