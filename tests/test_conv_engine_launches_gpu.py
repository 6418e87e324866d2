"""Every convolution launch the native engine makes, checked one by one against oracle/conv_desc.py at the benchmark's
shapes: c2 (480p, 5 objects) and c3 (1080p, 16 objects).

The engine (deva/model/native_engine.py on the synthetic checkpoint) runs encode_image, transform_key, encode_mask and
one decode with the sensory update, on the inputs test_engine_float64_gpu.py makes (config-1 frames, soft masks).
``deva._native.conv2d`` is wrapped: before each launch the stream is synchronised and the oracle evaluates the launch's
descriptor on the inputs as they stand then (so nothing the launch or a later one writes can change them); after it,
the outputs are compared element by element and only the statistics are kept.  Launches of fewer than 2^16 output
pixels are evaluated whole; larger ones on a sample: every pixel of the first and last row and column of the first and
last image, one full row and one full column of tile boundaries (flat tiles: both ends of every 128-pixel run) and 4096
seeded random pixels, widened to whole 4x4 windows where the launch pools.  Each launch is named by its weights
(``w_packed.data_ptr()`` in ``engine.P``).

Bound per element of a chain of n_k k-iterations (e4m3 ones included) and magnitude M (the oracle's sum of |term|):
    |f32 - exact| <= (4 n_k + 8) 2^-23 M
a model of wgmma's accumulator rounding toward zero at every step, not a measured constant; tools/accum_probe.py's
5e-5 of max |ref| at 216 k-iterations is consistent with it.  fp16 / e4m3 outputs must be the exact conversions of the
launch's own f32 where it writes f32; otherwise they lie within the same bound plus half an ulp of the output type.
The fused head, the 4x4 pool and the gated update carry that bound through their own arithmetic (see ``_bounds``).
A row per launch is printed: layer, b x h x w, cin -> cout, tile, channel tile, epilogue form, ksplit, mode and the
worst err / bound.
"""
import inspect
import os
import sys
import time

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_engine_float64_gpu as tef  # noqa: E402  (the inputs of the float64 engine check)

from oracle import conv_desc as cd  # noqa: E402

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -23
WHOLE = 1 << 16   # launches with fewer output pixels are evaluated whole
N_RANDOM = 4096


def _hulp(x, mant):
    """Half an ulp of |x| in a format with `mant` explicit mantissa bits (fp16: 10, e4m3: 3), and at least half its
    smallest subnormal spacing."""
    _, e = torch.frexp(x.abs().double())
    sub = {10: 2.0 ** -25, 3: 2.0 ** -10}[mant]
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), e - mant - 2).clamp_min(sub)


def _staged(kw):
    """Whether the launch takes the staged epilogue (conv.cu plan_staged; DEVA_B200_CONV_EPI unset)."""
    nt, n_mma = kw['nt'], min(w for w in (64, 128, 192, 256) if w >= kw['nt'])
    if kw.get('gate_out') is not None or kw.get('ksplit', 0) > 1 or kw.get('out_f32') is not None or nt != n_mma \
            or kw['cout'] != kw['cout_pad']:
        return False
    used = [kw.get('out_raw') is not None or kw.get('out_pool4') is not None] + \
        [kw.get(k) is not None for k in ('out_raw_lo', 'out_relu', 'out_relu_lo')]
    if kw.get('out_relu_lo8') is not None:
        return max(sum(used), 1 if kw.get('res') is not None else 0, 2 if kw.get('res_lo') is not None else 0) <= 2
    return sum(used) <= 3


def _mode(kw):
    m = ['x2' if kw.get('x2') is not None else 'x_lo' if kw.get('x_lo') is not None else
         {2: 'w_lo', 3: 'lo8'}.get(kw.get('split_mode', 0), 'plain')]
    for key, tag in (('rank1_w', 'rank1'), ('res', 'res'), ('res_lo', 'res_lo'), ('head_w', 'head'),
                     ('out_pool4', 'pool4'), ('gate_out', 'gates')):
        if kw.get(key) is not None:
            m.append(tag)
    if kw.get('res_broadcast'):
        m.append('bcast')
    return '+'.join(m)


def _sample(kw, ho, wo, seed):
    """Flat output-pixel indices to evaluate (None: all of them)."""
    b = kw['batch']
    if b * ho * wo < WHOLE:
        return None
    dev = kw['x'].device
    ys, xs = torch.arange(ho, device=dev), torch.arange(wo, device=dev)
    parts = []
    for img in sorted({0, b - 1}):
        base = img * ho * wo
        parts += [base + y * wo + xs for y in (0, ho - 1)] + [base + ys * wo + x for x in (0, wo - 1)]
    if kw['th'] == 0:  # flat tiles: both ends of every 128-pixel run of image 0
        p = torch.arange(ho * wo, device=dev)
        parts.append(p[(p % 128 == 0) | (p % 128 == 127)])
    else:
        th, tw = kw['th'], kw['tw']
        parts += [y * wo + xs for y in (th - 1, th) if y < ho] + [ys * wo + x for x in (tw - 1, tw) if x < wo]
    g = torch.Generator(device=dev).manual_seed(seed)
    parts.append(torch.randint(b * ho * wo, (N_RANDOM,), generator=g, device=dev))
    pix = torch.unique(torch.cat(parts))
    if kw.get('out_pool4') is not None:  # whole 4x4 windows
        img, y, x = pix // (ho * wo), pix // wo % ho // 4 * 4, pix % wo // 4 * 4
        d = torch.arange(4, device=dev)
        pix = torch.unique((img * ho * wo + y * wo + x).view(-1, 1, 1) + d.view(1, 4, 1) * wo + d.view(1, 1, 4))
    return pix


def _bounds(o, kw):
    """[(output name, got, exact, bound)] over the evaluated pixels (float64)."""
    b, cout = kw['batch'], kw['cout']
    n = b * o.ho * o.wo
    pix = o.pix
    nk = torch.tensor(o.nk, dtype=torch.float64, device=pix.device).view(-1, 1, 1)
    chain_bound = (4 * nk + 8) * EPS * o.chain_mag                       # [chains, P, cout]
    bound = chain_bound.sum(0)
    v = o.value
    rows = []

    def out(name, width=cout, count=n):
        buf = kw[name]
        return torch.as_strided(buf, (count * width,), (1,), buf.storage_offset()).view(count, width)

    f32 = None
    if kw.get('out_f32') is not None:
        parts = len(o.chains)
        f32 = torch.as_strided(kw['out_f32'], (parts * n * cout,), (1,), kw['out_f32'].storage_offset()) \
            .view(parts, n, cout)[:, pix]
        rows.append(('f32', f32.double(), o.chain_value, chain_bound))
    conv = cd.convert(f32[0]) if f32 is not None and len(o.chains) == 1 else None
    a = v.clamp_min(0)
    for name, exact in (('raw', v), ('relu', a)):
        key = 'out_' + name
        if kw.get(key) is None:
            continue
        got = out(key)[pix]
        lo = out(key + '_lo')[pix] if kw.get(key + '_lo') is not None else None
        if conv is not None:  # exact conversions of the launch's own f32
            for nm, gt in ((name, got), (name + '_lo', lo)):
                if gt is not None:
                    same = gt.view(torch.int16) == conv[nm].view(torch.int16)
                    rows.append((nm + ' = cvt(f32)', (~same).double(), torch.zeros_like(v), torch.zeros_like(v)))
        if lo is None:
            rows.append((name, got.double(), exact, bound + _hulp(torch.maximum(got.double().abs(), exact.abs()), 10)))
        else:
            rows.append((name + '+' + name + '_lo', got.double() + lo.double(), exact, bound + 2 * _hulp(lo.double(), 10)))
    if kw.get('out_relu_lo8') is not None:
        lo8 = cd.e4m3_to_f64(out('out_relu_lo8')[pix])
        if conv is not None:
            same = out('out_relu_lo8')[pix] == conv['relu_lo8']
            rows.append(('relu_lo8 = cvt(f32)', (~same).double(), torch.zeros_like(v), torch.zeros_like(v)))
        hi = out('out_relu')[pix].double()
        rows.append(('relu+relu_lo8', hi + lo8 / 4096, a, bound + _hulp(lo8, 3) / 4096))
    if kw.get('head_w') is not None:
        hn = kw['head_n']
        hw = kw['head_w'].double().view(hn, cout)
        got = out('head_out', hn)[pix].double()
        hb = bound @ hw.abs().t() + (cout / 4 + 3) * EPS * o.outputs['head_mag']
        rows.append(('head', got, o.outputs['head'], hb))
    if kw.get('out_pool4') is not None:
        win = o.outputs['pool4_win']
        q = pix
        wid = (q // (o.ho * o.wo) * (o.ho // 4) + q // o.wo % o.ho // 4) * (o.wo // 4) + q % o.wo // 4
        order = torch.argsort(wid, stable=True)
        sel = torch.isin(wid[order], win)
        idx = order[sel]
        ev = v[idx].view(-1, 16, cout)
        pb = (bound[idx] + _hulp(v[idx], 10)).view(-1, 16, cout).mean(1) + 16 * EPS * ev.abs().mean(1)
        exact = ev.mean(1)
        got = out('out_pool4', count=n // 16)[win].double()
        rows.append(('pool4', got, exact, pb + _hulp(exact, 10)))
    if kw.get('gate_out') is not None:
        c = cout // 3
        got = out('gate_out', c)[pix].double()
        bb = bound.view(-1, c // 64, 3, 64)
        hp = o.outputs['gate_h'].view(-1, c // 64, 64).abs()
        gb = (0.25 * hp * bb[:, :, 0] + 0.25 * (hp + 1) * bb[:, :, 1] + bb[:, :, 2]).reshape(-1, c)
        gb = gb + 2e-6 * (1 + o.outputs['gate_h'].abs()) + _hulp(o.outputs['gate'], 10)
        rows.append(('gate', got, o.outputs['gate'], gb))
    return rows


class Recorder:
    """The conv2d wrapper: oracle before, comparison after, one row of statistics per launch.  ``check=False`` records
    the launch descriptors only (no oracle, pixels and worst 0)."""

    def __init__(self, engine, real, check=True):
        self.names = {pc.w_packed.data_ptr(): name for name, pc in engine.P.items()}
        self.nt_packed = {name: pc.nt for name, pc in engine.P.items()}
        self.real, self.sig = real, inspect.signature(real)
        self.rows, self.stage, self.check = [], '', check

    def __call__(self, *args, **kwargs):
        ba = self.sig.bind(*args, **kwargs)
        ba.apply_defaults()
        kw = dict(ba.arguments)
        name = self.names.get(kw['w_packed'].data_ptr(), '?')
        pad = kw['kh'] // 2
        ho, wo = (kw['h'] + 2 * pad - kw['kh']) // kw['stride'] + 1, (kw['w'] + 2 * pad - kw['kh']) // kw['stride'] + 1
        if not self.check:
            self.real(**kw)
            self._row(kw, name, 0, 0.0, '')
            return
        torch.cuda.synchronize()
        o = cd.launch(pixels=_sample(kw, ho, wo, len(self.rows)), **kw)
        self.real(**kw)
        torch.cuda.synchronize()
        worst, where = 0.0, ''
        for what, got, exact, bnd in _bounds(o, kw):
            err = (got - exact).abs()
            ratio = torch.where(err == 0, torch.zeros_like(err), err / bnd)
            ratio = torch.where(torch.isnan(got), torch.full_like(err, float('inf')), ratio)
            r = float(ratio.max())
            if not r <= worst:
                i = int(ratio.reshape(-1).argmax())
                per = got.shape[-1]
                chain, rest = divmod(i, got[0].numel()) if got.dim() == 3 else (0, i)
                p, ch = divmod(rest, per)
                loc = f'{what} chain {chain} channel {ch}'
                if what == 'pool4':
                    loc += f' window {int(o.outputs["pool4_win"][p])}'
                else:
                    q = int(o.pix[p])
                    loc += f' image {q // (ho * wo)} y {q // wo % ho} x {q % wo}'
                worst, where = r, f'{loc}: |err| {float(err.reshape(-1)[i]):.3e}, bound {float(bnd.reshape(-1)[i]):.3e}'
        self._row(kw, name, o.pix.numel(), worst, where)

    def _row(self, kw, name, pixels, worst, where):
        self.rows.append(dict(
            stage=self.stage, layer=name, shape=f"{kw['batch']}x{kw['h']}x{kw['w']}",
            chans=f"{kw['cin_pad']}->{kw['cout']}", tile='flat' if kw['th'] == 0 else f"{kw['th']}x{kw['tw']}",
            nt=kw['nt'], narrowed=name in self.nt_packed and kw['nt'] < self.nt_packed[name],
            epi='staged' if _staged(kw) else 'regs', ksplit=max(kw.get('ksplit', 0), 1), mode=_mode(kw),
            pixels=pixels, worst=worst, where=where))


def run_stages(engine, rec, frames, masks, chunk_size=-1):
    """encode_image (frame 0), transform_key, encode_mask from a zero sensory state, encode_image (frame 1) and one
    decode with the sensory update, with ``rec.stage`` naming the stage of every launch.  Returns the decode's
    (sensory, logits)."""
    k = masks.shape[1]
    rec.stage = 'encode_image'
    ms, feat = engine.encode_image(frames[0:1])
    rec.stage = 'transform_key'
    engine.transform_key(feat)
    rec.stage = 'encode_mask'
    hh, ww = ms[0].shape[-2:]
    zero = torch.zeros(1, k, engine.value_dim, hh, ww, dtype=torch.float16, device='cuda')
    value, sensory = engine.encode_mask(frames[0:1], ms, zero, masks, chunk_size=chunk_size)
    rec.stage = 'encode_image'
    ms1, _ = engine.encode_image(frames[1:2])
    rec.stage = 'decode'
    return engine.decode(ms1, value, sensory, masks, chunk_size=chunk_size)


def report(case, rows, seconds):
    """Print one row per launch, then assert that every launch met its bound and was named."""
    print(f'\n{case}: {len(rows)} convolution launches checked in {seconds:.1f} s')
    print(f"    {'stage':13s} {'layer':44s} {'b x h x w':13s} {'cin->cout':10s} {'tile':6s} {'nt':>4s} "
          f"{'epi':6s} {'ks':>2s} {'mode':24s} {'pixels':>7s} err/bound")
    for r in rows:
        print(f"    {r['stage']:13s} {r['layer']:44s} {r['shape']:13s} {r['chans']:10s} {r['tile']:6s} "
              f"{r['nt']:4d}{'*' if r['narrowed'] else ' '}{r['epi']:6s} {r['ksplit']:2d} {r['mode']:24s} "
              f"{r['pixels']:7d} {r['worst']:.3f}")
    bad = [r for r in rows if not r['worst'] <= 1]
    assert not bad, '\n'.join(f"{r['layer']} ({r['stage']}, {r['mode']}): {r['where']}" for r in bad)
    assert all(r['layer'] != '?' for r in rows), 'a launch with weights outside engine.P'


@pytest.fixture(scope='module', autouse=True)
def _duration():
    t0 = time.perf_counter()
    yield
    print(f'\ntest_conv_engine_launches_gpu.py: {time.perf_counter() - t0:.1f} s')


@pytest.fixture(scope='module')
def engine(synthetic_sd):
    from deva.model.native_engine import NativeEngine
    from deva import _native
    _native.require_device()
    return NativeEngine({k: v.cuda() for k, v in synthetic_sd.items()})


@pytest.mark.parametrize('case', list(tef.CASES))
def test_every_launch_within_its_bound(case, engine, golden_dir, monkeypatch):
    from deva import _native as nat
    t0 = time.perf_counter()
    hw, k, _ = tef.CASES[case]
    frames = tef._frames(golden_dir, hw, 2)
    masks = tef._soft_masks(k, hw)
    rec = Recorder(engine, nat.conv2d)
    monkeypatch.setattr(nat, 'conv2d', rec)
    run_stages(engine, rec, frames, masks)
    monkeypatch.undo()
    torch.cuda.synchronize()
    rows = rec.rows
    report(case, rows, time.perf_counter() - t0)
    if case == 'c3':  # the paths only the large shapes reach: a change that stops reaching one must say so
        want = {
            'flat tiles': any(r['tile'] == 'flat' for r in rows),
            'a narrowed channel tile': any(r['narrowed'] for r in rows),
            'the pool4 + head launch': any('head' in r['mode'] and 'pool4' in r['mode'] for r in rows),
            'the gate launch': any('gates' in r['mode'] for r in rows),
            'an act_lo8 launch': any(r['mode'].startswith('lo8') for r in rows),
            'a split-K key launch': any(r['ksplit'] > 1 and r['layer'].startswith('key_proj') for r in rows),
        }
        missing = [k for k, ok in want.items() if not ok]
        assert not missing, f'c3 no longer reaches {missing}'
