"""Mint the wide top-k fixture by running the UNMODIFIED reference on CPU (build container only).

    python tests/golden/make_topk_golden.py

The 16-frame seeded clip and synthetic checkpoint of make_golden.golden_vos, at top_k = 50 and 100, on frames large
enough (160 x 192 -> 10 x 12 = 120 memory slots per frame) that the first read's window already holds more than
top_k slots.  Per top_k it records per-frame bank sizes, id maps and confident-pixel masks (top-2 probability gap > 0.05),
probabilities on the 4 x 4 pixel lattice [:, 1::4, 2::4] (as config1_vos does), and the similarity and the affinity of
the first memory read (do_softmax's input and output).  The frames are not stored: the test regenerates them from the
seed, and the fixture keeps their sum and absolute sum to prove it.  Writes topk_wide.{json,npz} next to this file.
"""
import json
import os
import sys

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_golden as mg  # noqa: E402  (the reference import shims)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import deva.inference.memory_manager as ref_mm  # noqa: E402  (the reference's module)

TOP_KS = (50, 100)
H, W, T = 160, 192, 16


def clip():
    g = torch.Generator().manual_seed(11)
    base = torch.randn(3, H, W, generator=g)
    frames = torch.stack([base + 0.2 * torch.randn(3, H, W, generator=g) for _ in range(T)])
    m0 = torch.zeros(H, W, dtype=torch.long); m0[12:80, 12:88] = 1; m0[88:152, 80:180] = 2
    m6 = torch.zeros(H, W, dtype=torch.long); m6[20:68, 112:184] = 7
    return frames, m0, m6


def run(top_k, frames, m0, m6):
    sd = mg.param_spec.synthetic_state_dict(seed=1)
    cfg = dict(mg.CFG, mem_every=1, max_long_term_elements=300, top_k=top_k)
    net = mg.DEVA(cfg).eval()
    net.load_weights(sd)
    np.random.seed(42)
    core = mg.DEVAInferenceCore(net, cfg)
    reads = []
    plain = ref_mm.do_softmax

    def spy(similarity, top_k=None, inplace=False, return_usage=False):
        sim = similarity.clone()
        out = plain(similarity, top_k=top_k, inplace=inplace, return_usage=return_usage)
        if not reads:
            reads.append((sim, (out[0] if return_usage else out).clone()))
        return out

    ref_mm.do_softmax = spy
    try:
        arrays, sizes = {}, []
        for t in range(T):
            if t == 0:
                p = core.step(frames[t], m0, [1, 2])
            elif t == 6:
                p = core.step(frames[t], m6, [7])
            else:
                p = core.step(frames[t], end=(t == T - 1))
            top2 = torch.topk(p, 2, dim=0)[0]
            arrays[f'prob_{t:02d}'] = p[:, 1::4, 2::4].contiguous()
            arrays[f'ids_{t:02d}'] = core.object_manager.tmp_to_obj_cls(torch.argmax(p, dim=0)).to(torch.uint8)
            arrays[f'confident_{t:02d}'] = torch.from_numpy(np.packbits(((top2[0] - top2[1]) > 0.05).numpy()))
            mem = core.memory
            sizes.append({str(b): [mem.work_mem.size(b), mem.long_mem.size(b)] for b in mem.work_mem.buckets})
    finally:
        ref_mm.do_softmax = plain
    sim, aff = reads[0]
    arrays['read_sim'], arrays['read_aff'] = sim[0], aff[0]  # [N, Q]
    print(f'  top_k {top_k}: first read N = {sim.shape[1]}, Q = {sim.shape[2]}; final sizes {sizes[-1]}')
    return cfg, sizes, {f'k{top_k}_{k}': v for k, v in arrays.items()}


def main():
    frames, m0, m6 = clip()
    meta = {'top_ks': list(TOP_KS), 'configs': {}, 'sizes': {}, 'frames_sum': float(frames.double().sum()),
            'frames_abs_sum': float(frames.double().abs().sum())}
    arrays = dict(mask0=m0.to(torch.uint8), mask6=m6.to(torch.uint8))
    for top_k in TOP_KS:
        cfg, sizes, a = run(top_k, frames, m0, m6)
        meta['configs'][str(top_k)], meta['sizes'][str(top_k)] = cfg, sizes
        arrays.update(a)
    mg.HERE = os.path.dirname(os.path.abspath(__file__))
    mg.save('topk_wide.npz', **arrays)
    json.dump(meta, open(os.path.join(mg.HERE, 'topk_wide.json'), 'w'))


if __name__ == '__main__':
    main()
