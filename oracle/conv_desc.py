"""Oracle: float64 semantics of one ``deva_b200_conv2d`` launch, read from its descriptor alone.

``launch(**kw)`` takes the keyword arguments of ``deva._native.conv2d`` (tensors plus the shape fields) and returns what
that launch must compute, in float64 on the operands' device.  It is written from the descriptor contract
(include/deva_b200.h, csrc/conv.cu) and reads each operand the way the kernel does: ``n`` contiguous elements from the
tensor's first element, whatever shape or strides the caller's tensor has.

* Passes over the fp16 operands (w_packed = [cout_pad, w_groups, taps, cin_pad]):
  plain X.W0;  x2: X.W0 + X2.W1;  split_mode 2: X.Wh + X.Wl;  x_lo: Xh.Wh + Xl.Wh + Xh.Wl.
  split_mode 3 adds Xlo8.W8 over the e4m3 bytes of x_lo8 and w8_packed ([cout_pad, taps * cin_pad]), and the whole
  accumulator is multiplied by acc_scale.  Padding is k // 2; stride 2 samples the same NHWC buffer.
* k-iterations are numbered as the kernel's producer issues them: the e4m3 entries first (one per tap and 128-channel
  block), then the fp16 entries t = pass * taps + tap, each in 64-channel blocks cb.  ksplit > 1 cuts them into chains
  of ceil(k_iters / ksplit); empty trailing chains do not exist.  Only chain 0 adds the bias.
* Epilogue terms, in the kernel's order: bias, rank1_w[ch] * rank1_x[pix], res, res_lo (batch stride 0 when
  res_broadcast).
* Outputs are conversions of the fp32 value (``convert``), the fused head relu(v) . head_w^T, the 4x4 pool of the raw
  fp16 output, and the gated update f * h * (1 - u) + u * tanh(n) over the packed [f | u | n] x 64 channel tiles.

Every value comes with its magnitude M: the sum of |product| over every term that enters the element (times
|acc_scale|), plus |bias|, |rank-1 term|, |res| and |res_lo|.  Error bounds are built from M.  ``pixels`` evaluates a
subset of the output pixels (flat indices into [batch, ho, wo]): a gather of their im2col rows and one float64 matmul
per chain.
"""
import math
from typing import Dict, List, Optional, Tuple

import torch

E4M3_MAX = 448.0
_CHUNK_ELEMS = 1 << 23  # float64 im2col elements per pixel chunk (64 MB)


def _stored(t: torch.Tensor, shape, dtype) -> torch.Tensor:
    """The kernel's view of ``t``: prod(shape) contiguous elements from its first element."""
    assert t.dtype == dtype, (t.dtype, dtype)
    n = math.prod(shape)
    return torch.as_strided(t, (n,), (1,), t.storage_offset()).view(*shape)


def e4m3_to_f64(u8: torch.Tensor) -> torch.Tensor:
    return u8.view(torch.float8_e4m3fn).to(torch.float32).double()


def f64_to_e4m3(v: torch.Tensor) -> torch.Tensor:
    """Round to nearest e4m3, saturating at +-448 (cvt.rn.satfinite): uint8 bytes."""
    return v.float().clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)


def convert(v32: torch.Tensor) -> Dict[str, torch.Tensor]:
    """The epilogue's conversions of fp32 values: raw / raw_lo, relu / relu_lo (fp16 of what the rounding dropped) and
    relu_lo8 = e4m3((a - fp16(a)) * 4096) of a = relu(v)."""
    assert v32.dtype == torch.float32
    raw = v32.half()
    a = v32.clamp_min(0)
    relu = a.half()
    return dict(raw=raw, raw_lo=(v32 - raw.float()).half(), relu=relu, relu_lo=(a - relu.float()).half(),
                relu_lo8=f64_to_e4m3((a - relu.float()) * 4096))


class Launch:
    """What one launch computes on ``pix`` (flat output-pixel indices into [batch, ho, wo]).

    chains [(k0, k1)]: k-iteration range of each chain;  nk [n_chains]: its length
    chain_value / chain_mag [n_chains, P, cout] float64 (chain 0 carries the bias and the epilogue terms)
    value / mag [P, cout]: their sums;  mag8 [P, cout]: sum |x8 * w8| in accumulator units (split_mode 3), else None
    outputs: dict name -> expected output on ``pix`` (see ``launch``)"""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def _passes(kw) -> Tuple[List[Tuple[str, int]], int]:
    """[(activation source, weight group)] of the fp16 passes, and w_groups."""
    x2, x_lo, sm = kw.get('x2'), kw.get('x_lo'), kw.get('split_mode', 0)
    if x2 is not None and x_lo is not None:
        raise ValueError('x2 and x_lo are exclusive')
    if sm not in (0, 2, 3):
        raise ValueError(f'split_mode {sm} unknown')
    if sm == 2:
        if x2 is not None or x_lo is not None:
            raise ValueError('split_mode 2 takes a single input')
        return [('x', 0), ('x', 1)], 2
    if sm == 3 and (x2 is not None or x_lo is not None or kw.get('x_lo8') is None or kw.get('w8_packed') is None
                    or kw['stride'] != 1 or kw['cin_pad'] % 128 or kw.get('ksplit', 0) > 1):
        raise ValueError('split_mode 3 needs x_lo8 + w8_packed, stride 1, cin_pad % 128 == 0, no x_lo / x2 / ksplit')
    if x2 is not None:
        return [('x', 0), ('x2', 1)], 2
    if x_lo is not None:
        return [('x', 0), ('x_lo', 0), ('x', 1)], 2
    return [('x', 0)], 1


def k_layout(kw) -> Tuple[int, int, List[Tuple[int, int]]]:
    """(k8, k_iters, chains): e4m3 k-iterations, all k-iterations, [(k0, k1)] of each non-empty chain."""
    kt = kw['kh'] * kw['kh']
    passes, _ = _passes(kw)
    k8 = kt * (kw['cin_pad'] // 128) if kw.get('split_mode', 0) == 3 else 0
    k_iters = k8 + len(passes) * kt * (kw['cin_pad'] // 64)
    ksplit = max(kw.get('ksplit', 0), 1)
    if ksplit > k_iters:
        raise ValueError(f'ksplit {ksplit} exceeds the {k_iters} k-iterations')
    per = -(-k_iters // ksplit)
    return k8, k_iters, [(k0, min(k_iters, k0 + per)) for k0 in range(0, k_iters, per)]


def launch(pixels: Optional[torch.Tensor] = None, **kw) -> Launch:
    """Float64 semantics of ``nat.conv2d(**kw)`` on the output pixels ``pixels`` (all when None).

    outputs: 'f32' [n_chains, P, cout] fp32 when out_f32 is wanted (one entry per chain); 'raw', 'raw_lo', 'relu',
    'relu_lo', 'relu_lo8' [P, cout] as ``convert`` of the fp32 value, when wanted; 'head' [P, head_n] float64 and
    'head_mag' (sum |relu(v) * head_w|); 'gate' [P, cout / 3] float64 with 'gate_h' (the previous state, float64);
    'pool4' [windows, cout] fp16 for the 4x4 windows all of whose pixels are in ``pixels``, at flat window indices
    'pool4_win' into [batch, ho / 4, wo / 4]."""
    b, h, w, cin_pad, kh, stride = (kw[k] for k in ('batch', 'h', 'w', 'cin_pad', 'kh', 'stride'))
    cout, cout_pad = kw['cout'], kw['cout_pad']
    if kh not in (1, 3) or stride not in (1, 2) or cin_pad % 64:
        raise ValueError('unsupported filter / stride / cin_pad')
    pad, taps = kh // 2, kh * kh
    ho, wo = (h + 2 * pad - kh) // stride + 1, (w + 2 * pad - kh) // stride + 1
    passes, w_groups = _passes(kw)
    k8, k_iters, chains = k_layout(kw)
    acc_scale = kw.get('acc_scale', 0.0) or 1.0
    if kw.get('gate_out') is not None and acc_scale != 1.0:
        raise ValueError('the gate epilogue takes an unscaled accumulator (acc_scale 0 or 1)')
    dev = kw['x'].device
    if pixels is None:
        pixels = torch.arange(b * ho * wo, device=dev)
    pix = pixels.to(dev, torch.long)

    # operands as stored, and the columns of each k-iteration: e4m3 entries (128 per k-iteration) then fp16 (64)
    srcs = {name: _stored(kw[name], (b, h, w, cin_pad), torch.float16) for name in ('x', 'x2', 'x_lo')
            if kw.get(name) is not None}
    wp = _stored(kw['w_packed'], (cout_pad, w_groups, taps, cin_pad), torch.float16)
    entries = []  # (source, tap, weight rows [cout, cin_pad] float64)
    if k8:
        srcs['x_lo8'] = _stored(kw['x_lo8'], (b, h, w, cin_pad), torch.uint8)
        w8 = e4m3_to_f64(_stored(kw['w8_packed'], (cout_pad, taps, cin_pad), torch.uint8)[:cout])
        entries += [('x_lo8', t, w8[:, t]) for t in range(taps)]
    for src, group in passes:
        entries += [(src, t, wp[:cout, group, t].double()) for t in range(taps)]
    wmat = torch.cat([e[2] for e in entries], 1).t().contiguous()  # [K, cout]
    wabs = wmat.abs()

    def col(ki):  # first im2col column of k-iteration ki
        return ki * 128 if ki < k8 else k8 * 128 + (ki - k8) * 64

    bias = _stored(kw['bias'], (cout_pad,), torch.float32)[:cout].double()
    rank1 = None
    if kw.get('rank1_w') is not None:
        rank1 = (_stored(kw['rank1_w'], (cout_pad,), torch.float32)[:cout].double(),
                 _stored(kw['rank1_x'], (b * ho * wo,), torch.float32).double())
    rb = 1 if kw.get('res_broadcast') else b
    res = [_stored(kw[k], (rb, ho * wo, cout), torch.float16) for k in ('res', 'res_lo') if kw.get(k) is not None]
    if kw.get('res_lo') is not None and kw.get('res') is None:
        raise ValueError('res_lo needs res')

    n_ch = len(chains)
    cv = torch.empty(n_ch, pix.numel(), cout, dtype=torch.float64, device=dev)
    cm = torch.empty_like(cv)
    mag8 = torch.empty(pix.numel(), cout, dtype=torch.float64, device=dev) if k8 else None
    step = max(1, _CHUNK_ELEMS // wmat.shape[0])
    for p0 in range(0, pix.numel(), step):
        pc = pix[p0:p0 + step]
        bi, yo, xo = pc // (ho * wo), pc // wo % ho, pc % wo
        cols = []
        for src, t, _ in entries:
            yi, xi = yo * stride + t // kh - pad, xo * stride + t % kh - pad
            ok = (yi >= 0) & (yi < h) & (xi >= 0) & (xi < w)
            rows = srcs[src][bi, yi.clamp(0, h - 1), xi.clamp(0, w - 1)]
            rows = e4m3_to_f64(rows) if src == 'x_lo8' else rows.double()
            cols.append(rows * ok.unsqueeze(1))
        a = torch.cat(cols, 1)
        aabs = a.abs()
        for c, (k0, k1) in enumerate(chains):
            s = slice(col(k0), col(k1))
            cv[c, p0:p0 + step] = (a[:, s] @ wmat[s]) * acc_scale
            cm[c, p0:p0 + step] = (aabs[:, s] @ wabs[s]) * abs(acc_scale)
        if k8:
            mag8[p0:p0 + step] = aabs[:, :k8 * 128] @ wabs[:k8 * 128]
        del a, aabs, cols

    # epilogue terms (chain 0)
    cv[0] += bias
    cm[0] += bias.abs()
    if rank1 is not None:
        term = rank1[0].unsqueeze(0) * rank1[1][pix].unsqueeze(1)
        cv[0] += term
        cm[0] += term.abs()
    if res:
        rbat = pix // (ho * wo) if rb == b else torch.zeros_like(pix)
        for r in res:
            term = r[rbat, pix % (ho * wo)].double()
            cv[0] += term
            cm[0] += term.abs()
    value, mag = cv.sum(0), cm.sum(0)

    outs = {}
    if kw.get('out_f32') is not None:
        outs['f32'] = cv.float()
    conv = convert(value.float())
    for name in ('raw', 'raw_lo', 'relu', 'relu_lo', 'relu_lo8'):
        if kw.get('out_' + name) is not None:
            outs[name] = conv[name]
    if kw.get('head_w') is not None:
        hw = _stored(kw['head_w'], (kw['head_n'], cout), torch.float32).double()
        a = value.clamp_min(0)
        outs['head'], outs['head_mag'] = a @ hw.t(), a @ hw.abs().t()
    if kw.get('gate_out') is not None:
        if kw.get('nt') != 192 or cout % 192 or cout != cout_pad:
            raise ValueError('the gate epilogue needs nt 192 and cout = cout_pad = 3 * C, C % 64 == 0')
        c = cout // 3
        g = value.view(-1, c // 64, 3, 64)
        f, u, n = torch.sigmoid(g[:, :, 0]), torch.sigmoid(g[:, :, 1]), torch.tanh(g[:, :, 2])
        hp = _stored(kw['gate_h'], (b * ho * wo, c), torch.float16)[pix].double().view(-1, c // 64, 64)
        outs['gate'] = (f * hp * (1 - u) + u * n).reshape(-1, c)
        outs['gate_h'] = hp.reshape(-1, c)
    if kw.get('out_pool4') is not None:
        if ho % 4 or wo % 4:
            raise ValueError('out_pool4 needs ho, wo multiples of 4')
        win = (pix // (ho * wo) * (ho // 4) + pix // wo % ho // 4) * (wo // 4) + pix % wo // 4
        wins, count = torch.unique(win, return_counts=True)
        full = wins[count == 16]
        sel = torch.isin(win, full)
        order = torch.argsort(win[sel], stable=True)
        raw = conv['raw'][sel][order].double().view(-1, 16, cout)
        outs['pool4'] = (raw.sum(1) / 16).half()
        outs['pool4_win'] = full
    return Launch(pix=pix, ho=ho, wo=wo, chains=chains, nk=[k1 - k0 for k0, k1 in chains], k8=k8, k_iters=k_iters,
                  chain_value=cv, chain_mag=cm, value=value, mag=mag, mag8=mag8, outputs=outs)
