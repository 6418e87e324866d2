"""Stage-by-stage GPU parity of the native network kernels against the reference-minted per-stage fixture
(tests/golden/network_stages.npz: encode_image, transform_key, encode_mask, segment of the UNMODIFIED reference on one
64x80 frame with two objects).  Every stage gets the FIXTURE's inputs, so a regression shows up in the stage that owns
it instead of as a clip-level drift.  The measured errors are printed; the bounds are all tighter than what a single wrong
layer produces (> 1e-1)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    assert tuple(a.shape) == tuple(b.shape), (a.shape, b.shape)
    err = float((a - b).abs().max())
    return err, err / max(float(b.abs().max()), 1e-30)


def test_native_engine_stages_match_reference(golden_dir, synthetic_sd):
    from deva.model.native_engine import NativeEngine
    g = {k: torch.from_numpy(v).cuda() for k, v in np.load(os.path.join(golden_dir, 'network_stages.npz')).items()}
    eng = NativeEngine({k: v.cuda() for k, v in synthetic_sd.items()})
    report = {}

    # ---- key encoder (split precision): a10, a11
    ms, feat = eng.encode_image(g['image'])
    for name, got, want in (('f16', ms[0], g['f16']), ('f8', ms[1], g['f8']), ('f4', ms[2], g['f4']), ('feat', feat, g['feat'])):
        report[name] = _rel(got, want)
        assert report[name][1] < 8e-4, (name, report[name])  # fp16 storage of a ~fp32 result: 2^-11 of the largest value
    key, shr, sel = eng.transform_key(feat)
    for name, got, want, tol in (('key', key, g['key'], 3e-4), ('shrinkage', shr, g['shrinkage'], 3e-4),
                                 ('selection', sel, g['selection'], 5e-5)):
        report[name] = _rel(got, want)
        assert report[name][0] < tol, (name, report[name])

    # ---- value encoder on the fixture's state (a13); multi-scale features: the engine's own (they carry the lo parts)
    value, s1 = eng.encode_mask(g['image'], ms, g['sensory0'].half(), g['masks'])
    report['value'] = _rel(value, g['value'])
    report['sensory1'] = _rel(s1, g['sensory1'])
    assert report['value'][1] < 2.5e-3, report['value']
    assert report['sensory1'][0] < 8e-3, report['sensory1']

    # ---- decoder on the fixture's readout / sensory / masks (a12), then the output tail (a14)
    s2, logits = eng.decode(ms, g['readout'], g['sensory1'].half(), g['masks'])
    report['sensory2'] = _rel(s2, g['sensory2'])
    full, prob = eng.probabilities(logits.float().contiguous(), want_logits=True)
    report['logits'] = _rel(full, g['logits'])
    report['prob'] = _rel(prob, g['prob'])
    torch.cuda.synchronize()
    print('stage errors (max abs, relative to max |ref|):')
    for k, (e, r) in report.items():
        print(f'    {k:10s} {e:.3e}  {r:.3e}')
    assert report['sensory2'][0] < 2e-2, report['sensory2']
    assert report['logits'][0] < 8e-3, report['logits']
    assert report['prob'][0] < 1e-3, report['prob']
