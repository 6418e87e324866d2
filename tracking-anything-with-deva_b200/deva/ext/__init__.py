"""Detector-facing helpers of the demos (API of the reference's deva/ext/).

This package provides ``automatic_sam`` and ``grounding_dino``: the step that turns a detector's mask stack into the
detection id map runs on the device.  Everything else under ``deva.ext`` (``SAM``, ``MobileSAM``, ``LightHQSAM``,
``ext_eval_args``, ``automatic_processor``, ``with_text_processor``) resolves to the reference checkout when one is on
sys.path after this package, and the reference's processors pick up these functions unchanged.
"""
from pkgutil import extend_path

__path__ = extend_path(__path__, __name__)
