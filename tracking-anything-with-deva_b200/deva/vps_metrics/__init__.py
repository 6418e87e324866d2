"""VIPSeg video panoptic metrics (VPQ, STQ) and stuff merging on the device, drop-in for the reference's
``deva.vps_metrics``: ``eval_vpq_vipseg.eval_vpq``, ``eval_stq_vipseg.eval_stq`` and ``stuff_merging.merge_stuff`` keep
their signatures and read and write the same files; ``eval_vps`` writes both metrics' files from one decode pass.
Importing the package does not initialise CUDA."""
# Modules this package does not provide resolve to the reference checkout when one is on sys.path after this package.
from pkgutil import extend_path

__path__ = extend_path(__path__, __name__)


def eval_vps(submit_dir, truth_dir, pan_gt_json_file, num_processes=None, *, png_decoder=None):
    from deva.vps_metrics.video_pass import eval_vps as run
    return run(submit_dir, truth_dir, pan_gt_json_file, num_processes, png_decoder=png_decoder)
