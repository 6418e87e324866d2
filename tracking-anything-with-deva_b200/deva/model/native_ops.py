"""Host-side wrappers of the sm_90a network kernels: weight packing, tile choice, op calls.

Activations are fp16 NHWC torch tensors [B, H, W, C]; weights are packed once per checkpoint into the
layout the implicit-GEMM kernel streams with TMA ([Cout_pad, taps * Cin_pad] fp16, BN folded bias fp32).
"""
import os
from typing import Optional, Tuple

import torch

from deva import _native as nat

CBAM_POOL_SPLIT = 64  # csrc/elementwise.cu kPoolSplit: pixel slices of the CBAM channel pooling (scratch layout)
MAX_CHAIN = 32  # longest single accumulation chain of a split-precision conv (k-iterations of 64 channels)
CHAIN = 27      # chain length when a longer loop is split (= one 3x3 filter over 64 channels in three passes)
PROFILE = None  # set to a list by bench.py to collect (start event, end event, algorithmic FLOPs, MMA passes) per conv

_TILES = ((1, 128), (2, 64), (4, 32), (8, 16), (16, 8), (32, 4))
FLAT = (0, 128)  # flat tiles: 128 consecutive output pixels of one image (stride 1, no pool4)
FLAT_TILES = True  # False: rectangles only (tools/bench_conv.py --rect compares the two)
NT_WIDTHS = (256, 192, 128, 64)  # channel tiles with a wgmma width of their own (the staged epilogue takes exactly these)


def choose_tile(ho: int, wo: int, pool4: bool = False, stride: int = 1) -> Tuple[int, int]:
    """(th, tw) with th*tw = 128 that wastes the fewest MMA rows on an ho x wo output (``pool4``: among the tiles
    whose sides are multiples of 4, which the epilogue's 4x4 pooling needs).  A stride-1 launch without ``pool4`` takes
    flat tiles (``FLAT``) when they waste strictly fewer rows than the best rectangle, e.g. at 68 x 120 (1/16 of 1080p),
    where (1, 128) computes 68 tiles for 63.75 tiles of pixels.  The tile does not change any result."""
    best, best_cost = None, None
    for th, tw in _TILES:
        if pool4 and (th % 4 or tw % 4):
            continue
        cost = -(-ho // th) * th * (-(-wo // tw) * tw)
        if best_cost is None or cost < best_cost or (cost == best_cost and tw > best[1]):
            best, best_cost = (th, tw), cost
    if FLAT_TILES and stride == 1 and not pool4 and -(-ho * wo // 128) * 128 < best_cost:
        return FLAT
    return best


def pixel_tiles(ho: int, wo: int, tile: Tuple[int, int]) -> int:
    """Pixel tiles of one ho x wo image under ``tile`` (th, tw), flat or rectangular."""
    th, tw = tile
    return -(-ho * wo // 128) if th == 0 else -(-ho // th) * -(-wo // tw)


def choose_nt(nt: int, cout_pad: int, m_tiles: int, ksplit: int, sms: int) -> int:
    """Channel tile of one launch.  The kernel's persistent CTAs take work units (pixel tile, channel tile, k-split) in
    waves of ``sms``; a unit costs about its width, so a launch costs ~ ceil(units / sms) * width.  Of ``nt`` (the
    packed default) and the narrower widths in NT_WIDTHS that divide ``cout_pad`` this returns the cheapest, ties to the
    wider.  A narrower tile must save more than 1/8: it re-reads the activation tile and runs one more epilogue per
    pixel tile, which the model leaves out, so launches of four or more waves keep ``nt``.  A ``nt`` outside NT_WIDTHS
    (a ragged tile) stays.  A batch-1 1/16-resolution layer with 256 channels is 64 pixel tiles: one
    256-wide wave on 64 SMs, or one 128-wide wave on 128.  No width changes any result: every output element takes the
    same k-iterations in the same order."""
    if nt not in NT_WIDTHS:
        return nt
    ksplit = max(ksplit, 1)

    def cost(w):
        return -(-m_tiles * (cout_pad // w) * ksplit // sms) * w
    best, base = nt, cost(nt)
    for w in NT_WIDTHS:  # widest first: a tie keeps the wider
        if w < nt and cout_pad % w == 0 and 8 * cost(w) < 7 * base and cost(w) < cost(best):
            best = w
    return best


_SMS = {}


def _sm_count(dev) -> int:
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    if idx not in _SMS:
        _SMS[idx] = torch.cuda.get_device_properties(idx).multi_processor_count
    return _SMS[idx]


def _round_up(x, m):
    return (x + m - 1) // m * m


class PackedConv:
    """One convolution ready for ``deva_b200_conv2d``."""
    def __init__(self, weight: torch.Tensor, bias: Optional[torch.Tensor], stride: int,
                 rank1_in: Optional[int] = None, two_inputs: bool = False, precise: bool = False,
                 gates: bool = False, w_lo: bool = False, act_lo8: bool = False,
                 nt_override: Optional[int] = None):
        """weight [Cout, Cin, k, k] fp32 (BN folded); if ``rank1_in`` is given, that input channel is split
        off as a rank-1 term (out += w[:, rank1_in] * x1) - used for the '+1' mask / logit channels.
        ``gates``: Cout = [forget | update | new] x C of a sensory updater; rows are regrouped so that every
        192-channel tile holds the three gates of 64 hidden channels and the conv epilogue applies the update.
        Precision modes (exclusive): ``precise`` = inputs (hi, lo) x weights (hi, lo), three MMA passes, ~fp32;
        ``w_lo`` = single fp16 input x weights (hi, lo), two passes (no weight rounding);
        ``act_lo8`` = fp16 inputs plus a low-order pass on the fp8 path (no activation-operand rounding): the activation
        remainder arrives as e4m3 of (x - fp16(x)) * 4096, the weights are packed twice - fp16(W * 2^S) and
        e4m3(W * 2^(S-12)) - and the epilogue scales the common accumulator by 2^-S; the correction pass covers 128
        channels per k-iteration, i.e. costs half a pass."""
        cout, cin, kh, kw = weight.shape
        self.gates = gates
        if gates:
            c_hidden = cout // 3
            assert cout == 3 * c_hidden and c_hidden % 64 == 0
            order = torch.arange(cout, device=weight.device).view(3, c_hidden // 64, 64).permute(1, 0, 2).reshape(-1)
            weight = weight[order]
            bias = bias[order] if bias is not None else None
        assert kh == kw and kh in (1, 3)
        dev = weight.device
        self.rank1_w = None
        if rank1_in is not None:
            assert kh == 1
            keep = [c for c in range(cin) if c != rank1_in]
            r1 = weight[:, rank1_in, 0, 0].float()
            weight = weight[:, keep]
            cin -= 1
        self.two_inputs = two_inputs
        self.precise = precise  # split precision: weights stored as fp16 (hi, lo), inputs arrive as (hi, lo)
        self.w_lo, self.act_lo8 = w_lo, act_lo8
        assert int(precise) + int(w_lo) + int(act_lo8) <= 1 and not (two_inputs and (precise or w_lo or act_lo8))
        self.split_mode = 2 if w_lo else (3 if act_lo8 else 0)
        self.takes_lo = precise
        self.takes_lo8 = act_lo8
        self.w8_packed, self.acc_scale = None, 0.0
        if two_inputs:  # the layer consumes cat[x, x2]: pack [cout, source, tap, cin/2]
            assert cin % 128 == 0 and stride == 1
            cin //= 2
        self.cout, self.cin, self.k, self.stride = cout, cin, kh, stride
        self.cin_pad = _round_up(cin, 64)
        if gates:
            self.nt = 192
        elif cout >= 256:
            self.nt = 256 if cout % 256 == 0 else (128 if cout % 128 == 0 else 0)
        else:
            self.nt = _round_up(cout, 32)
        if self.nt == 0:
            self.nt = 256
        self.nt_fixed = gates  # the gate epilogue takes 192-wide tiles only
        if nt_override is not None:  # channel-tile experiments (tools/bench_conv.py)
            assert not gates and nt_override % 32 == 0 and 32 <= nt_override <= 256
            self.nt = nt_override
            self.nt_fixed = True
        self.cout_pad = _round_up(cout, self.nt)
        nsrc = 2 if two_inputs else 1
        w = torch.zeros(self.cout_pad, nsrc, kh * kw, self.cin_pad, dtype=torch.float32, device=dev)
        for s_ in range(nsrc):
            part = weight[:, s_ * cin:(s_ + 1) * cin]
            w[:cout, s_, :, :cin] = part.permute(0, 2, 3, 1).reshape(cout, kh * kw, cin)
        if precise or w_lo:
            hi = w.half()
            lo = (w - hi.float()).half()
            w = torch.cat([hi.float(), lo.float()], 1)
            nsrc = 2
        if act_lo8:
            assert self.cin_pad % 128 == 0 and stride == 1, 'the fp8 correction pass needs Cin % 128 == 0 and stride 1'
            import math
            s_exp = math.floor(math.log2(60000.0 / max(float(w.abs().max()), 1e-30)))
            self.acc_scale = 2.0 ** (-s_exp)
            self.w8_packed = (w * 2.0 ** (s_exp - 12)).reshape(self.cout_pad, kh * kw * self.cin_pad) \
                .to(torch.float8_e4m3fn).view(torch.uint8).contiguous()
            w = w * 2.0 ** s_exp
        self.w_packed = w.reshape(self.cout_pad, nsrc * kh * kw * self.cin_pad).half().contiguous()
        self.bias = torch.zeros(self.cout_pad, dtype=torch.float32, device=dev)
        if bias is not None:
            self.bias[:cout] = bias.float()
        if rank1_in is not None:
            self.rank1_w = torch.zeros(self.cout_pad, dtype=torch.float32, device=dev)
            self.rank1_w[:cout] = r1

    def to(self, device) -> 'PackedConv':
        """Packing runs where the checkpoint lives (the engine packs on the host); this uploads the packed operands."""
        self.w_packed = self.w_packed.to(device)
        self.bias = self.bias.to(device)
        if self.w8_packed is not None:
            self.w8_packed = self.w8_packed.to(device)
        if self.rank1_w is not None:
            self.rank1_w = self.rank1_w.to(device)
        return self

    def out_hw(self, h: int, w: int) -> Tuple[int, int]:
        p = self.k // 2
        return (h + 2 * p - self.k) // self.stride + 1, (w + 2 * p - self.k) // self.stride + 1


class ConvOut:
    __slots__ = ('raw', 'raw_lo', 'relu', 'relu_lo', 'relu_lo8', 'f32', 'head', 'hidden', 'pool4')

    def __init__(self):
        self.raw = self.raw_lo = self.relu = self.relu_lo = self.relu_lo8 = self.f32 = self.head = self.hidden = None
        self.pool4 = None


def conv_ex(x: torch.Tensor, pc: PackedConv, *, x2: Optional[torch.Tensor] = None, x_lo: Optional[torch.Tensor] = None,
            res: Optional[torch.Tensor] = None, res_lo: Optional[torch.Tensor] = None,
            rank1_x: Optional[torch.Tensor] = None, want_raw: bool = False, want_relu: bool = False,
            want_f32: bool = False, want_lo: bool = False, head_w: Optional[torch.Tensor] = None,
            gate_h: Optional[torch.Tensor] = None, ksplit: int = 0, x_lo8: Optional[torch.Tensor] = None,
            want_relu_lo8: bool = False, want_pool4: bool = False) -> ConvOut:
    """x fp16 NHWC [B,H,W,cin_pad] (+ x2: implicit channel concat, or + x_lo: split precision) -> ConvOut.
    ``want_pool4``: ``pool4`` = area_down(raw, 4), pooled in the epilogue without writing ``raw`` unless it is wanted too."""
    if want_pool4 and os.environ.get('DEVA_B200_CONV_EPI') == 'regs':  # the per-thread epilogue cannot pool (A/B runs)
        o = conv_ex(x, pc, x2=x2, x_lo=x_lo, res=res, res_lo=res_lo, rank1_x=rank1_x, want_raw=True, want_relu=want_relu,
                    want_f32=want_f32, want_lo=want_lo, head_w=head_w, gate_h=gate_h, ksplit=ksplit, x_lo8=x_lo8,
                    want_relu_lo8=want_relu_lo8)
        o.pool4 = area_down(o.raw, 4)
        if not want_raw:
            o.raw = o.raw_lo = None
        return o
    assert x.dtype == torch.float16 and x.is_contiguous() and x.shape[-1] == pc.cin_pad, (x.shape, pc.cin_pad)
    assert (x2 is not None) == pc.two_inputs and (x_lo is not None) == pc.takes_lo, (x_lo is None, pc.takes_lo)
    assert (x_lo8 is not None) == pc.takes_lo8
    if x_lo8 is not None:
        assert x_lo8.dtype == torch.uint8 and x_lo8.is_contiguous() and x_lo8.shape == x.shape
    for other in (x2, x_lo):
        if other is not None:
            assert other.dtype == torch.float16 and other.is_contiguous() and other.shape == x.shape
    b, h, w, _ = x.shape
    ho, wo = pc.out_hw(h, w)
    th, tw = choose_tile(ho, wo, want_pool4, pc.stride)
    dev = x.device

    def new(dtype=torch.float16):
        return torch.empty(b, ho, wo, pc.cout, dtype=dtype, device=dev)

    # Split-precision layers keep at most MAX_CHAIN k-iterations in one accumulator: the tensor core rounds toward
    # zero at every accumulation step, and a deep K loop (3x3 x 256 channels x 3 passes = 108 k-iterations) leaves a
    # systematic relative error that the top-k read downstream of the key path does not tolerate
    # (tools/accum_probe.py measures it).  Longer loops run as chains of <= CHAIN k-iterations
    # whose fp32 partial sums are added - with the bias, the residual and the output conversions - by sum_parts.
    k_iters = pc.k * pc.k * (pc.cin_pad // 64) * (3 if pc.precise else (2 if (pc.w_lo or pc.two_inputs) else 1))
    if (pc.precise and ksplit == 0 and k_iters > MAX_CHAIN and not (want_f32 or want_pool4 or head_w is not None or pc.rank1_w is not None)
            and pc.cout % 8 == 0 and (res is None or res.shape[0] == b)):
        parts = conv_ex(x, pc, x_lo=x_lo, want_f32=True, ksplit=-(-k_iters // CHAIN)).f32
        o = ConvOut()
        if want_raw:
            o.raw = torch.empty(b, ho, wo, pc.cout, dtype=torch.float16, device=dev)
            o.raw_lo = torch.empty_like(o.raw) if want_lo else None
        if want_relu:
            o.relu = torch.empty(b, ho, wo, pc.cout, dtype=torch.float16, device=dev)
            o.relu_lo = torch.empty_like(o.relu) if want_lo else None
        nat.sum_parts(parts, parts.shape[0], parts[0].numel(), parts[0].numel(), res=res, res_lo=res_lo, raw=o.raw,
                      raw_lo=o.raw_lo, relu=o.relu, relu_lo=o.relu_lo)
        return o
    o = ConvOut()
    if want_raw:
        o.raw = new()
        o.raw_lo = new() if want_lo else None
    if want_relu:
        o.relu = new()
        o.relu_lo = new() if want_lo else None
        o.relu_lo8 = new(torch.uint8) if want_relu_lo8 else None
    if want_pool4:
        o.pool4 = torch.empty(b, ho // 4, wo // 4, pc.cout, dtype=torch.float16, device=dev)
    if want_f32:
        o.f32 = new(torch.float32)
        if ksplit > 1:  # fp32 partial sums [parts, b, ho, wo, cout] of a split K loop; the consumer adds them
            k_iters = pc.k * pc.k * (pc.cin_pad // 64) * (3 if pc.precise else (2 if (pc.w_lo or pc.two_inputs) else 1))
            per = -(-k_iters // ksplit)
            o.f32 = torch.empty(-(-k_iters // per), b, ho, wo, pc.cout, dtype=torch.float32, device=dev)
    res_b = False
    if res is not None:
        assert res.dtype == torch.float16 and res.is_contiguous() and res.shape[1:] == (ho, wo, pc.cout)
        res_b = res.shape[0] == 1 and b > 1
        assert res_b or res.shape[0] == b
        assert res_lo is None or (res_lo.shape == res.shape and res_lo.is_contiguous())
    if pc.rank1_w is not None:
        assert rank1_x is not None and rank1_x.dtype == torch.float32 and rank1_x.numel() == b * ho * wo
    head_n = 0
    if head_w is not None:  # fused 1x1 head on relu(result): [head_n, cout] fp32
        head_n = head_w.shape[0]
        assert head_w.dtype == torch.float32 and head_w.is_contiguous() and head_w.shape[1] == pc.cout
        o.head = torch.empty(b, ho, wo, head_n, dtype=torch.float32, device=dev)
    assert (gate_h is not None) == pc.gates
    if gate_h is not None:  # fused hidden-state update: the conv output itself is never written
        assert gate_h.dtype == torch.float16 and gate_h.is_contiguous() and gate_h.shape == (b, ho, wo, pc.cout // 3)
        assert not (want_raw or want_relu or want_f32 or res is not None or head_w is not None)
        o.hidden = torch.empty_like(gate_h)
    if PROFILE is not None:  # bench.py's conv-roofline pass: CUDA events around the launch + algorithmic FLOPs
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
    nt = pc.nt
    if not (pc.nt_fixed or head_w is not None):  # the head needs the whole Cout in one tile
        nt = choose_nt(pc.nt, pc.cout_pad, b * pixel_tiles(ho, wo, (th, tw)), ksplit, _sm_count(dev))
    nat.conv2d(x, b, h, w, pc.cin_pad, pc.w_packed, pc.k, pc.stride, pc.cout, pc.cout_pad, nt, th, tw, pc.bias,
               x2=x2, x_lo=x_lo, res=res, res_lo=res_lo, res_broadcast=res_b, rank1_w=pc.rank1_w,
               rank1_x=rank1_x if pc.rank1_w is not None else None, out_raw=o.raw, out_relu=o.relu, out_f32=o.f32,
               out_raw_lo=o.raw_lo, out_relu_lo=o.relu_lo, head_w=head_w, head_out=o.head, head_n=head_n,
               gate_h=gate_h, gate_out=o.hidden, split_mode=pc.split_mode, ksplit=ksplit, x_lo8=x_lo8,
               w8_packed=pc.w8_packed, acc_scale=pc.acc_scale, out_relu_lo8=o.relu_lo8, out_pool4=o.pool4)
    if PROFILE is not None:
        ev1.record()
        flops = 2.0 * b * ho * wo * pc.cout * pc.k * pc.k * pc.cin * (2 if pc.two_inputs else 1)
        PROFILE.append((ev0, ev1, flops, 3 if pc.precise else (2 if pc.w_lo else (1.5 if pc.act_lo8 else 1))))
    return o


def conv(x: torch.Tensor, pc: PackedConv, *, x2: Optional[torch.Tensor] = None, res: Optional[torch.Tensor] = None,
         rank1_x: Optional[torch.Tensor] = None, want_raw: bool = False, want_relu: bool = False,
         want_f32: bool = False):
    """Plain-precision convenience form: returns the requested outputs (raw fp16, relu fp16, raw fp32) as a tuple
    (or the single tensor)."""
    o = conv_ex(x, pc, x2=x2, res=res, rank1_x=rank1_x, want_raw=want_raw, want_relu=want_relu, want_f32=want_f32)
    outs = tuple(t for t in (o.raw, o.relu, o.f32) if t is not None)
    return outs[0] if len(outs) == 1 else outs


def pack_stem(weight: torch.Tensor, bias: Optional[torch.Tensor], precise: bool = False) -> PackedConv:
    """7x7 stride-2 stem weights [64, C, 7, 7] -> a 1x1 PackedConv over the im2col columns (kh, kw, c)."""
    cout, cin, kh, kw = weight.shape
    assert kh == 7 and kw == 7
    cols = weight.permute(0, 2, 3, 1).reshape(cout, kh * kw * cin, 1, 1)
    return PackedConv(cols, bias, 1, precise=precise)


def stem_columns(planes: torch.Tensor, k_pad: int, with_lo: bool = False):
    """fp32 planes [B, C, H, W] -> fp16 im2col [B, H/2, W/2, k_pad] (and its fp16 remainder) for the 7x7 stride-2 stem."""
    b, c, h, w = planes.shape
    out = torch.empty(b, h // 2, w // 2, k_pad, dtype=torch.float16, device=planes.device)
    lo = torch.empty_like(out) if with_lo else None
    nat.stem_im2col(planes.contiguous(), out, b, c, h, w, k_pad, dst_lo=lo)
    return (out, lo) if with_lo else out


def maxpool(x: torch.Tensor, x_lo: Optional[torch.Tensor] = None):
    b, h, w, c = x.shape
    y = torch.empty(b, (h + 1) // 2, (w + 1) // 2, c, dtype=torch.float16, device=x.device)
    y_lo = torch.empty_like(y) if x_lo is not None else None
    nat.maxpool(x, y, b, h, w, c, x_lo=x_lo, y_lo=y_lo)
    return (y, y_lo) if x_lo is not None else y


def up2_add_split(g: torch.Tensor, g_lo: torch.Tensor, skip: torch.Tensor, skip_lo: torch.Tensor,
                  want_relu_lo8: bool = False):
    """(g + g_lo) bilinear x2 + (skip + skip_lo) -> (raw, raw_lo, relu, relu_lo8): the residual stream stays a fp16
    hi/lo pair; relu_lo8 (the e4m3 remainder of relu) only when the consumer runs the fp8 correction pass."""
    b, h, w, c = g.shape
    assert skip.shape == (1, 2 * h, 2 * w, c) and g_lo.shape == g.shape and skip_lo.shape == skip.shape
    new = lambda: torch.empty(b, 2 * h, 2 * w, c, dtype=torch.float16, device=g.device)  # noqa: E731
    raw, raw_lo, relu = new(), new(), new()
    relu_lo8 = torch.empty(b, 2 * h, 2 * w, c, dtype=torch.uint8, device=g.device) if want_relu_lo8 else None
    nat.up2_add_split(g, g_lo, skip, raw, raw_lo, relu, b, h, w, c, skip_lo=skip_lo, relu_lo8=relu_lo8)
    return raw, raw_lo, relu, relu_lo8


def area_down(x: torch.Tensor, r: int) -> torch.Tensor:
    b, h, w, c = x.shape
    y = torch.empty(b, h // r, w // r, c, dtype=torch.float16, device=x.device)
    nat.area_down(x, y, b, h, w, c, r)
    return y


def area_down_plane(x: torch.Tensor, r: int) -> torch.Tensor:
    """fp32 [B,H,W] -> [B,H/r,W/r]"""
    b, h, w = x.shape
    y = torch.empty(b, h // r, w // r, dtype=torch.float32, device=x.device)
    nat.area_down_plane(x.contiguous(), y, b, h, w, r)
    return y


def cbam_residual_split(x: torch.Tensor, x_lo: torch.Tensor, params: dict):
    """(x + x_lo) + CBAM(x + x_lo) -> (raw, raw_lo, relu) on fp16 NHWC; params: w1,b1,w2,b2 (channel MLP), ws [2*49],
    bs [1] (fp32)."""
    b, h, w, c = x.shape
    r = params['w1'].shape[0]
    scratch = torch.empty((2 * CBAM_POOL_SPLIT + 1) * b * c + 2 * b * h * w, dtype=torch.float32, device=x.device)
    raw, raw_lo, relu = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    nat.cbam_split(x, x_lo, params['w1'], params['b1'], params['w2'], params['b2'], params['ws'], params['bs'], scratch,
                   raw, raw_lo, relu, b, h, w, c, r)
    return raw, raw_lo, relu
