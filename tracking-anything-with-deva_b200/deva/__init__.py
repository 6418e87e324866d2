"""Drop-in ``deva`` package: DEVA's propagation API on H100-native kernels.

Same import surface as the reference (deva/__init__.py:1-2): ``deva.DEVAInferenceCore`` and
``deva.DEVA``.  Imports are lazy so that pure-host modules (checkpoint spec, object bookkeeping)
stay importable on machines without a GPU.
"""
# Modules this package does not provide (dataset readers, result savers, detectors, training code, ...) resolve to the
# reference checkout when one is on sys.path *after* this package: same-named package directories are chained,
# ours first (pkgutil.extend_path), so `evaluation/eval_vos.py` and `deva/ext/*` import unchanged.
from pkgutil import extend_path

__path__ = extend_path(__path__, __name__)



def __getattr__(name):
    if name == 'DEVAInferenceCore':
        from deva.inference.inference_core import DEVAInferenceCore
        return DEVAInferenceCore
    if name == 'DEVA':
        from deva.model.network import DEVA
        return DEVA
    raise AttributeError(name)
