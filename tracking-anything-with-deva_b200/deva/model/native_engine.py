"""The DEVA propagation network on the hand-written sm_90a kernels (NHWC fp16, wgmma implicit GEMM).

Same forward graphs as ``oracle/network.py`` (which restates the reference's network.py /
big_modules.py / modules.py / group_modules.py / cbam.py / resnet.py), with BatchNorm folded and the
shared halves hoisted by ``LayerTable``; every layer is a ``deva_b200_conv2d`` launch with its bias / residual /
ReLU / rank-1 input fused in the epilogue, and the glue (max-pool, bilinear x2 + skip, area pooling,
CBAM, GRU gates, soft aggregation + x4 upsampling + softmax) runs in the helper kernels of
csrc/elementwise.cu.  No cuDNN / cuBLAS on this path.

Tensors crossing the public API keep the reference's [B, C, H, W] / [1, K, C, h, w] *shapes* but are
permuted views of NHWC fp16 storage, so they flow through ``DEVAInferenceCore`` / ``MemoryManager``
without conversion.  The key path, the decoder's residual stream and the layers next to the logits run at more than
fp16 precision (the precision plan in ``NativeEngine.__init__``), which keeps the probabilities within 1e-3 of fp32.
"""
from typing import Dict

import torch

from deva import _native as nat
from deva.model import native_ops as ops
from deva.model.layer_table import LayerTable

KEY_KSPLIT = 8  # accumulation chains of the key projection (see transform_key)


def _to_nhwc(t: torch.Tensor) -> torch.Tensor:
    """API tensor [B,C,H,W] (any strides / dtype) -> contiguous fp16 [B,H,W,C]; free for our own views."""
    x = t.permute(0, 2, 3, 1)
    if x.dtype == torch.float16 and x.is_contiguous():
        return x
    if t.dtype == torch.float32 and t.is_contiguous():
        b, c, h, w = t.shape
        out = torch.empty(b, h, w, c, dtype=torch.float16, device=t.device)
        nat.nchw_to_nhwc(t, out, b, c, h, w, c)
        return out
    return x.contiguous().half()


def _api(t_nhwc: torch.Tensor) -> torch.Tensor:
    return t_nhwc.permute(0, 3, 1, 2)


class NativeEngine:
    precision = 'parity'  # the name of the precision plan below, reported in bench.py's result line

    def __init__(self, sd: Dict[str, torch.Tensor]):
        # Precision plan (DESIGN "precision plan"; tools/precision_layers.py / precision_plan.py rank the rounding sources):
        # the decoder's residual / skip stream travels as fp16 (hi, lo) pairs, the 1x1 shortcut / skip convolutions that
        # consume the raw stream run in split precision (three MMA passes, they are cheap), sensory_compress takes (hi, lo)
        # weights, and the two 3x3 convs of the last decoder block (up_8_4, next to the logits) add an fp8 correction pass
        # over their activations' low-order part (half a pass).  max |prob - fp32 reference| < 1e-3.
        self.device = next(iter(sd.values())).device
        # fold BatchNorm and pack the operands on the host (a few hundred tiny device launches otherwise), upload once
        t = LayerTable({k: v.detach().to('cpu', torch.float32) if v.is_floating_point() else v.cpu() for k, v in sd.items()})
        self.key_dim, self.value_dim = t.key_dim, t.value_dim
        L = t.layers
        P: Dict[str, ops.PackedConv] = {}
        for name, spec in L.items():
            # The key path (pixel encoder -> key projection) runs in split precision (fp16 hi/lo pairs, ~fp32
            # accuracy): the top-k read is discontinuous in the keys, and the path is < 3 % of the frame's FLOPs.
            precise = name.startswith('pixel_encoder') or name.startswith('key_proj')
            tail = name.rsplit('.', 1)[-1]
            if tail in ('skip8', 'skip4', 'ds_x', 'ds_g') or name.endswith('up_16_8.out_conv.ds'):
                precise = True
            act_lo8 = 'up_8_4.out_conv' in name  # the low-order activation pass on the fp8 path
            w_lo = name.endswith('.sensory_compress')
            if name.endswith('.pred'):  # folded into up_8_4.c2's epilogue as a fp32 9-tap head (see decode)
                self.pred_w = spec.weight[0].permute(1, 2, 0).reshape(9, -1).float().contiguous().to(self.device)  # [tap, cin]
                self.pred_b = float(spec.bias[0])
                continue
            if name.endswith('.stem'):
                P[name] = ops.pack_stem(spec.weight, spec.bias, precise=True)
            elif name.endswith('.stem_img') or name.endswith('.stem_mask'):
                P[name] = ops.pack_stem(spec.weight, spec.bias)
            elif name.endswith('.gru'):
                P[name] = ops.PackedConv(spec.weight, spec.bias, 1, two_inputs=True, gates=True)
            else:
                rank1 = spec.weight.shape[1] - 1 if (name.endswith('.sensory_compress') or name.endswith('.su.g4_conv')) else None
                P[name] = ops.PackedConv(spec.weight, spec.bias, spec.stride, rank1_in=rank1, precise=precise,
                                         act_lo8=act_lo8, w_lo=w_lo)
        self.P = {k: v.to(self.device) for k, v in P.items()}
        self.cbam = {}
        for p, c in t.cbam.items():
            self.cbam[p] = {k: v.to(self.device) for k, v in dict(
                w1=c['w1'].contiguous(), b1=c['b1'].contiguous(), w2=c['w2'].contiguous(), b2=c['b2'].contiguous(),
                ws=c['ws'].reshape(-1).contiguous(), bs=c['bs'].contiguous()).items()}

    # ------------------------------------------------------------------ key encoder (a10, a11), split precision
    def _bottleneck(self, x, q):
        """x = (hi, lo) post-ReLU pair -> (hi, lo) pair (resnet.py:78-114 with BN folded)."""
        P = self.P
        y = ops.conv_ex(x[0], P[q + '.c1'], x_lo=x[1], want_relu=True, want_lo=True)
        y = ops.conv_ex(y.relu, P[q + '.c2'], x_lo=y.relu_lo, want_relu=True, want_lo=True)
        if (q + '.ds') in P:
            s_ = ops.conv_ex(x[0], P[q + '.ds'], x_lo=x[1], want_raw=True, want_lo=True)
            short = (s_.raw, s_.raw_lo)
        else:
            short = x
        o = ops.conv_ex(y.relu, P[q + '.c3'], x_lo=y.relu_lo, res=short[0], res_lo=short[1], want_relu=True, want_lo=True)
        return o.relu, o.relu_lo

    def encode_image(self, image: torch.Tensor):
        """image fp32 [1,3,H,W] -> ((f16, f8, f4), key_feat) as API views of NHWC fp16 tensors."""
        P, p = self.P, 'pixel_encoder'
        stem = P[p + '.stem']
        cols, cols_lo = ops.stem_columns(image.float(), stem.cin_pad, with_lo=True)
        o = ops.conv_ex(cols, stem, x_lo=cols_lo, want_relu=True, want_lo=True)
        x = ops.maxpool(o.relu, o.relu_lo)
        feats = []
        for stage, blocks in (('res2', 3), ('layer2', 4), ('layer3', 6)):
            for i in range(blocks):
                x = self._bottleneck(x, f'{p}.{stage}.{i}')
            feats.append(x)
        f4, f8, f16 = feats
        o1 = ops.conv_ex(f16[0], P[p + '.proj1'], x_lo=f16[1], want_raw=True, want_relu=True, want_lo=True)
        o2 = ops.conv_ex(f16[0], P[p + '.proj2'], x_lo=f16[1], want_raw=True, want_lo=True)
        f16_api = _api(o1.raw)
        f16_api._b200_relu = o1.relu  # ReLU twin for the fusers' shared half (kept alive with the view)
        f16_api._b200_lo = o1.raw_lo  # low-order parts: the shortcut / skip convs of the parity plan consume them
        f16_api._b200_relu_lo = o1.relu_lo
        f8_api, f4_api = _api(f8[0]), _api(f4[0])
        f8_api._b200_lo, f4_api._b200_lo = f8[1], f4[1]
        key_feat = _api(o2.raw)
        key_feat._b200_lo = o2.raw_lo  # low-order part for the split-precision key projection
        return (f16_api, f8_api, f4_api), key_feat

    def transform_key(self, feat: torch.Tensor, need_sk=True, need_ek=True):
        x = _to_nhwc(feat)
        lo = getattr(feat, '_b200_lo', None)
        if lo is None:
            lo = torch.zeros_like(x)
        _, h, w, _ = x.shape
        pc = self.P['key_proj.all']
        # split-K: the projection's 3 x 9 x Cin/64 k-iterations run as KSPLIT short accumulation chains whose fp32 partial
        # sums key_tail adds on the CUDA cores.  One accumulator over the whole loop (round-toward-zero at every
        # step) leaves a systematic error in the keys that can flip near-tied top-k members (tools/accum_probe.py).
        y = ops.conv_ex(x, pc, x_lo=lo, want_f32=True, ksplit=KEY_KSPLIT).f32  # [parts,1,h,w,2*CK+1] fp32
        q, ck = h * w, self.key_dim
        key = torch.empty(q, ck, dtype=torch.float32, device=x.device)
        sel = torch.empty(q, ck, dtype=torch.float32, device=x.device)
        shr = torch.empty(q, dtype=torch.float32, device=x.device)
        nat.key_tail(y, pc.cout, q, ck, key, shr, sel, n_parts=y.shape[0], part_stride=y[0].numel())
        return (key.view(1, h, w, ck).permute(0, 3, 1, 2), shr.view(1, 1, h, w) if need_sk else None,
                sel.view(1, h, w, ck).permute(0, 3, 1, 2) if need_ek else None)

    # ------------------------------------------------------------------ shared blocks
    @staticmethod
    def _lo_of(x_api: torch.Tensor, like: torch.Tensor) -> torch.Tensor:
        """Low-order part riding on an API view (zeros when the tensor came from elsewhere, e.g. a user's own features)."""
        lo = getattr(x_api, '_b200_lo', None)
        if lo is None or lo.shape != like.shape:
            lo = torch.zeros_like(like)
        return lo

    def _C(self, name, x, lo=None, **kw) -> ops.ConvOut:
        """Conv `name` on (x, lo): the low-order part is consumed only when the layer's precision mode takes it."""
        pc = self.P[name]
        if pc.takes_lo8:  # `lo` is the e4m3 remainder (uint8)
            return ops.conv_ex(x, pc, x_lo8=lo if lo is not None else torch.zeros(x.shape, dtype=torch.uint8, device=x.device), **kw)
        if pc.takes_lo:
            return ops.conv_ex(x, pc, x_lo=lo if lo is not None else torch.zeros_like(x), **kw)
        return ops.conv_ex(x, pc, **kw)

    def _tl(self, name) -> bool:
        return self.P[name].takes_lo

    def _fuse(self, p, X, g_raw, g_lo, g_relu, g_relu_lo=None):
        """GroupFeatureFusionBlock (group_modules.py:133-152): the block's residual stream (shortcut, block outputs, CBAM
        residual) is carried as (hi, lo) pairs and the two 1x1 shortcut convs - they map the raw stream straight onto the
        output - run in split precision; every MMA operand gets its low-order part when its layer's mode takes one.
        X = the shared feature (raw, raw_lo, relu, relu_lo).  Returns the block output [K,h,w,C] as (raw, raw_lo)."""
        x_raw, x_lo, x_relu, x_relu_lo = X
        q = p + '.b1'
        sx = self._C(q + '.c1_x', x_relu, x_relu_lo, want_raw=True, want_lo=True)
        dx = self._C(q + '.ds_x', x_raw, x_lo, want_raw=True, want_lo=True)
        y = self._C(q + '.c1_g', g_relu, g_relu_lo, res=sx.raw, res_lo=sx.raw_lo, want_relu=True, want_lo=self._tl(q + '.c2'))
        short = self._C(q + '.ds_g', g_raw, g_lo, res=dx.raw, res_lo=dx.raw_lo, want_raw=True, want_lo=True)
        g = self._C(q + '.c2', y.relu, y.relu_lo, res=short.raw, res_lo=short.raw_lo, want_raw=True, want_lo=True)
        gr_raw, gr_lo, gr_relu = ops.cbam_residual_split(g.raw, g.raw_lo, self.cbam[p])
        y = self._C(p + '.b2.c1', gr_relu, want_relu=True, want_lo=self._tl(p + '.b2.c2'))
        out = self._C(p + '.b2.c2', y.relu, y.relu_lo, res=gr_raw, res_lo=gr_lo, want_raw=True, want_lo=True)
        return out.raw, out.raw_lo

    def _shared_quad(self, x_api: torch.Tensor):
        raw = _to_nhwc(x_api)
        relu = getattr(x_api, '_b200_relu', None)
        if relu is None:
            relu = torch.relu(raw)
        relu_lo = getattr(x_api, '_b200_relu_lo', None)
        return raw, self._lo_of(x_api, raw), relu, relu_lo

    def _gru(self, key, g, h):
        # 3x3 conv over cat[g, h] -> (forget, update, new) gates -> h' (modules.py:145-149,163-167), one kernel:
        # the gates are evaluated on the fp32 accumulators in the conv epilogue, the 3C-channel tensor is never stored
        return ops.conv_ex(g, self.P[key], x2=h, gate_h=h).hidden

    # ------------------------------------------------------------------ value encoder (a13)
    def _basic(self, x, q):
        P = self.P
        y = ops.conv(x, P[q + '.c1'], want_relu=True)
        short = ops.conv(x, P[q + '.ds'], want_raw=True) if (q + '.ds') in P else x
        return ops.conv(y, P[q + '.c2'], res=short, want_relu=True)

    def _basic_pair(self, x, lo, q):
        """BasicBlock on a post-ReLU (hi, lo) pair: returns the output pair."""
        y = self._C(q + '.c1', x, lo, want_relu=True, want_lo=self._tl(q + '.c2'))
        if (q + '.ds') in self.P:
            s_ = self._C(q + '.ds', x, lo, want_raw=True, want_lo=True)
            short, short_lo = s_.raw, s_.raw_lo
        else:
            short, short_lo = x, lo
        o = self._C(q + '.c2', y.relu, y.relu_lo, res=short, res_lo=short_lo, want_relu=True, want_lo=True)
        return o.relu, o.relu_lo

    def encode_mask(self, image, ms_features, sensory, masks, deep_update=True, chunk_size=-1):
        """image [1,3,H,W], sensory [1,K,C,h,w], masks [1,K,H,W] -> (value, sensory') as API views."""
        P, p = self.P, 'mask_encoder'
        k = masks.shape[1]
        step = k if chunk_size < 1 or chunk_size >= k else chunk_size
        img_pc, msk_pc = P[p + '.stem_img'], P[p + '.stem_mask']
        shared = ops.conv(ops.stem_columns(image.float(), img_pc.cin_pad), img_pc, want_raw=True)
        X = self._shared_quad(ms_features[0])
        h_all = _to_nhwc(sensory[0])
        planes = masks[0].float().contiguous().unsqueeze(1)  # [K,1,H,W]
        values, hiddens = [], []
        for i in range(0, k, step):
            cols = ops.stem_columns(planes[i:i + step], msk_pc.cin_pad)
            # single-fp16 trunk; its last block hands the fuser a (hi, lo) pair
            x = ops.conv(cols, msk_pc, res=shared, want_relu=True)
            x = ops.maxpool(x)  # ReLU and max-pool commute (quirk Q6)
            for stage in ('layer1', 'layer2', 'layer3'):
                for b in range(2):
                    if stage == 'layer3' and b == 1:
                        x, lo = self._basic_pair(x, None, f'{p}.{stage}.{b}')
                    else:
                        x = self._basic(x, f'{p}.{stage}.{b}')
            g16, _ = self._fuse(p + '.fuser', X, x, lo, x, lo)
            values.append(g16)
            if deep_update:
                hiddens.append(self._gru(p + '.gru', g16, h_all[i:i + step].contiguous()))
        value = values[0] if len(values) == 1 else torch.cat(values, 0)
        if deep_update:
            new_h = hiddens[0] if len(hiddens) == 1 else torch.cat(hiddens, 0)
            new_sensory = _api(new_h).unsqueeze(0)
        else:
            new_sensory = sensory
        return _api(value).unsqueeze(0), new_sensory

    # ------------------------------------------------------------------ decoder (a12)
    def decode(self, ms_features, readout, sensory, last_mask, update_sensory=True, chunk_size=-1):
        """readout/sensory [1,K,C,h,w], last_mask [1,K,H,W] -> (sensory', logits fp32 [1,K,H/4,W/4])."""
        P, p = self.P, 'mask_decoder'
        f16, f8, f4 = ms_features
        k = readout.shape[1]
        step = k if chunk_size < 1 or chunk_size >= k else chunk_size
        f8n, f4n = _to_nhwc(f8), _to_nhwc(f4)
        X = self._shared_quad(f16)
        s8 = self._C(p + '.skip8', f8n, self._lo_of(f8, f8n), want_raw=True, want_lo=True)
        s4 = self._C(p + '.skip4', f4n, self._lo_of(f4, f4n), want_raw=True, want_lo=True)
        skip8, skip8_lo, skip4, skip4_lo = s8.raw, s8.raw_lo, s4.raw, s4.raw_lo
        ro_all = _to_nhwc(readout[0])
        h_all = _to_nhwc(sensory[0])
        hh, ww = ro_all.shape[1:3]
        lm = last_mask[0].float().contiguous()
        assert lm.shape[-2] == 16 * hh and lm.shape[-1] == 16 * ww
        last = ops.area_down_plane(lm, 16)  # [K,h,w] fp32: the '+1' input channel of sensory_compress
        logits_all, hiddens = [], []
        for i in range(0, k, step):
            h = h_all[i:i + step].contiguous()
            c16 = self._C(p + '.sensory_compress', h, rank1_x=last[i:i + step].contiguous(),
                          res=ro_all[i:i + step].contiguous(), want_raw=True, want_relu=True, want_lo=True)
            p16, p16_lo = self._fuse(p + '.fuser', X, c16.raw, c16.raw_lo, c16.relu, c16.relu_lo)
            q = p + '.up_16_8.out_conv'
            g8_raw, g8_lo, g8_relu, _ = ops.up2_add_split(p16, p16_lo, skip8, skip8_lo)
            y = self._C(q + '.c1', g8_relu, want_relu=True, want_lo=self._tl(q + '.c2'))
            short = self._C(q + '.ds', g8_raw, g8_lo, want_raw=True, want_lo=True)
            o8 = self._C(q + '.c2', y.relu, y.relu_lo, res=short.raw, res_lo=short.raw_lo, want_raw=True, want_lo=True)
            p8 = o8.raw
            q = p + '.up_8_4.out_conv'
            g4_raw, g4_lo, g4_relu, g4_relu_lo8 = ops.up2_add_split(p8, o8.raw_lo, skip4, skip4_lo, want_relu_lo8=True)
            y4 = self._C(q + '.c1', g4_relu, g4_relu_lo8, want_relu=True, want_relu_lo8=True)
            # p4 = c2(...) + g4; the logit conv pred(relu(p4)) (big_modules.py:189-190) is folded in: the epilogue
            # emits the 9 per-tap dot products in fp32, a 3x3 gather finishes the convolution.  p4 itself is only
            # read 4x4-pooled by su.g4_conv, so the epilogue writes that pool instead of p4.
            o4 = self._C(q + '.c2', y4.relu, y4.relu_lo8, res=g4_raw, res_lo=g4_lo, want_pool4=update_sensory,
                         head_w=self.pred_w)
            logits = torch.empty(o4.head.shape[0], 4 * hh, 4 * ww, 1, dtype=torch.float32, device=o4.head.device)
            nat.head_gather3x3(o4.head, logits, self.pred_b, o4.head.shape[0], 4 * hh, 4 * ww)
            logits_all.append(logits)
            if update_sensory:
                g = ops.conv(p16, P[p + '.su.g16_conv'], want_raw=True)
                g = ops.conv(ops.area_down(p8, 2), P[p + '.su.g8_conv'], res=g, want_raw=True)
                g = ops.conv(o4.pool4, P[p + '.su.g4_conv'], res=g, want_raw=True,
                             rank1_x=ops.area_down_plane(logits.view(-1, 4 * hh, 4 * ww), 4))
                hiddens.append(self._gru(p + '.gru', g, h))
        logits = logits_all[0] if len(logits_all) == 1 else torch.cat(logits_all, 0)
        if update_sensory:
            new_h = hiddens[0] if len(hiddens) == 1 else torch.cat(hiddens, 0)
            new_sensory = _api(new_h).unsqueeze(0)
        else:
            new_sensory = sensory
        return new_sensory, logits.view(1, k, 4 * hh, 4 * ww)

    # ------------------------------------------------------------------ output tail (a14, quirk Q8)
    def probabilities(self, logits: torch.Tensor, want_logits: bool = False):
        """logits fp32 [1,K,h4,w4] -> prob [1,K+1,4*h4,4*w4] (and the up-sampled aggregated logits)."""
        _, k, h4, w4 = logits.shape
        dev = logits.device
        agg = torch.empty(k + 1, h4, w4, dtype=torch.float32, device=dev)
        prob = torch.empty(1, k + 1, 4 * h4, 4 * w4, dtype=torch.float32, device=dev)
        full = torch.empty_like(prob) if want_logits else None
        nat.output_tail(logits.contiguous(), agg, prob, full, k, h4, w4)
        return full, prob
