"""VPQ of VIPSeg at window sizes 1, 2, 4, 6, 8, 10 and 999 (the reference's deva/vps_metrics/eval_vpq_vipseg.py) from
one joint label histogram per frame: the PNGs are decoded once, not once per window size, and every window is the
difference of two prefix sums.  Writes vpq-{n}.txt and vpq-simple.txt byte for byte as the reference does."""
import os
import time

from deva.vps_metrics import video_pass


def eval_vpq(submit_dir, truth_dir, pan_gt_json_file, num_processes=None):
    """num_processes: host threads that decode PNGs (default: up to 16)."""
    output_dir = submit_dir
    if not os.path.isdir(submit_dir):
        print("%s doesn't exist" % submit_dir)
    start_all = time.time()
    vpq_stats, _, categories_list = video_pass.evaluate(submit_dir, truth_dir, pan_gt_json_file, stq=False,
                                                        num_threads=num_processes)
    video_pass.write_vpq(output_dir, vpq_stats, categories_list)
    print('==> All:', time.time() - start_all, 'sec')
