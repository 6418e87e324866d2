"""Inference engine for the DEVA propagation network: a flat, BN-folded layer table + forward graphs.

The reference builds the network as an ``nn.Module`` tree (deva/model/big_modules.py, modules.py,
group_modules.py, cbam.py, resnet.py) and runs every conv / BN / ReLU / interpolate as its own ATen
call.  The engine instead

* folds every eval-mode BatchNorm into the preceding bias-free convolution at load time
  (w' = w * g/sqrt(var+eps), b' = beta - mean * g/sqrt(var+eps));
* splits convolutions whose input is ``cat[shared image feature, per-object feature]`` into a
  once-per-frame shared half and a per-object half (SURVEY.md section 7, hard part 5): the 7x7 stem of the
  mask encoder (image 3ch shared / mask 1ch per object) and ``fuser.block1.{conv1,downsample}`` of both
  fusers (512 shared / 256|512 per object);
* expresses the forward passes against a small op set implemented by a backend.

Backends: ``TorchOps`` (cuDNN/cuBLAS through ATen, fp32 NCHW) is the interim implementation of the conv
stack while the hand-written NHWC wgmma implicit-GEMM kernels land layer by layer; it is library code
on the device, never a CPU path.  The memory read never goes through a backend - it is always the
sm_90a kernels in deva/inference/memory_manager.py.
"""
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

BN_EPS = 1e-5


class ConvSpec:
    """One folded convolution: weight [Cout,Cin,k,k], bias [Cout], stride, padding."""
    __slots__ = ('weight', 'bias', 'stride', 'pad')

    def __init__(self, weight, bias, stride=1, pad=0):
        self.weight, self.bias, self.stride, self.pad = weight, bias, stride, pad


def _fold(sd, conv: str, bn: Optional[str], stride: int, pad: int) -> ConvSpec:
    w = sd[conv + '.weight'].float()
    b = sd.get(conv + '.bias')
    b = torch.zeros(w.shape[0], device=w.device) if b is None else b.float()
    if bn is not None:
        scale = sd[bn + '.weight'].float() / torch.sqrt(sd[bn + '.running_var'].float() + BN_EPS)
        w = w * scale.view(-1, 1, 1, 1)
        b = (b - sd[bn + '.running_mean'].float()) * scale + sd[bn + '.bias'].float()
    return ConvSpec(w.contiguous(), b.contiguous(), stride, pad)


def _split_in(spec: ConvSpec, n_shared: int) -> Tuple[ConvSpec, ConvSpec]:
    """Split along input channels: (shared half carrying the bias, per-object half without bias)."""
    shared = ConvSpec(spec.weight[:, :n_shared].contiguous(), spec.bias, spec.stride, spec.pad)
    own = ConvSpec(spec.weight[:, n_shared:].contiguous(), None, spec.stride, spec.pad)
    return shared, own


class LayerTable:
    """All folded layers of one checkpoint, on one device."""
    def __init__(self, sd: Dict[str, torch.Tensor]):
        L: Dict[str, ConvSpec] = {}
        # ---- pixel encoder: ResNet-50 stem..layer3 (reference resnet.py:78-152, big_modules.py:23-51)
        p = 'pixel_encoder'
        L[p + '.stem'] = _fold(sd, p + '.conv1', p + '.bn1', 2, 3)
        for stage, blocks, stride in (('res2', 3, 1), ('layer2', 4, 2), ('layer3', 6, 2)):
            for i in range(blocks):
                q = f'{p}.{stage}.{i}'
                s = stride if i == 0 else 1
                L[q + '.c1'] = _fold(sd, q + '.conv1', q + '.bn1', 1, 0)
                L[q + '.c2'] = _fold(sd, q + '.conv2', q + '.bn2', s, 1)
                L[q + '.c3'] = _fold(sd, q + '.conv3', q + '.bn3', 1, 0)
                if (q + '.downsample.0.weight') in sd:
                    L[q + '.ds'] = _fold(sd, q + '.downsample.0', q + '.downsample.1', s, 0)
        L[p + '.proj1'] = _fold(sd, p + '.proj1', None, 1, 0)
        L[p + '.proj2'] = _fold(sd, p + '.proj2', None, 1, 0)
        # ---- key projection (modules.py:60-78): the three 3x3 heads share their input -> one conv
        kp = [_fold(sd, 'key_proj.' + n, None, 1, 1) for n in ('key_proj', 'd_proj', 'e_proj')]
        self.key_dim = kp[0].weight.shape[0]
        L['key_proj.all'] = ConvSpec(torch.cat([c.weight for c in kp], 0).contiguous(),
                                     torch.cat([c.bias for c in kp], 0).contiguous(), 1, 1)
        # ---- mask encoder: ResNet-18 stem..layer3 + fuser + deep GRU (big_modules.py:54-127)
        p = 'mask_encoder'
        stem = _fold(sd, p + '.conv1', p + '.bn1', 2, 3)
        L[p + '.stem_img'], L[p + '.stem_mask'] = _split_in(stem, 3)
        for stage, stride in (('layer1', 1), ('layer2', 2), ('layer3', 2)):
            for i in range(2):
                q = f'{p}.{stage}.{i}'
                s = stride if i == 0 else 1
                L[q + '.c1'] = _fold(sd, q + '.conv1', q + '.bn1', s, 1)
                L[q + '.c2'] = _fold(sd, q + '.conv2', q + '.bn2', 1, 1)
                if (q + '.downsample.0.weight') in sd:
                    L[q + '.ds'] = _fold(sd, q + '.downsample.0', q + '.downsample.1', s, 0)
        # the fusers see cat[f16 (pix_feat_dim channels, shared), per-object feature]: split at the checkpoint's own width
        pix_dim = sd['pixel_encoder.proj1.weight'].shape[0]
        self._fusion(L, sd, p + '.fuser', pix_dim)
        L[p + '.gru'] = _fold(sd, p + '.sensory_update.transform', None, 1, 1)
        # ---- mask decoder (big_modules.py:130-212)
        p = 'mask_decoder'
        self._fusion(L, sd, p + '.fuser', pix_dim)
        sc = _fold(sd, p + '.sensory_compress', None, 1, 0)
        L[p + '.sensory_compress'] = sc
        L[p + '.skip8'] = _fold(sd, p + '.decoder_feat_proc.transforms.0', None, 1, 0)
        L[p + '.skip4'] = _fold(sd, p + '.decoder_feat_proc.transforms.1', None, 1, 0)
        for up in ('up_16_8', 'up_8_4'):
            q = f'{p}.{up}.out_conv'
            L[q + '.c1'] = _fold(sd, q + '.conv1', None, 1, 1)
            L[q + '.c2'] = _fold(sd, q + '.conv2', None, 1, 1)
            if (q + '.downsample.weight') in sd:
                L[q + '.ds'] = _fold(sd, q + '.downsample', None, 1, 0)
        L[p + '.pred'] = _fold(sd, p + '.pred', None, 1, 1)
        for n in ('g16_conv', 'g8_conv', 'g4_conv'):
            L[f'{p}.su.{n}'] = _fold(sd, f'{p}.sensory_update.{n}', None, 1, 0)
        L[p + '.gru'] = _fold(sd, p + '.sensory_update.transform', None, 1, 1)
        self.layers = L
        self.cbam = {}
        for p in ('mask_encoder.fuser', 'mask_decoder.fuser'):
            a = p + '.attention'
            self.cbam[p] = dict(w1=sd[a + '.ChannelGate.mlp.1.weight'].float(), b1=sd[a + '.ChannelGate.mlp.1.bias'].float(),
                                w2=sd[a + '.ChannelGate.mlp.3.weight'].float(), b2=sd[a + '.ChannelGate.mlp.3.bias'].float(),
                                ws=sd[a + '.SpatialGate.spatial.conv.weight'].float(),
                                bs=sd[a + '.SpatialGate.spatial.conv.bias'].float())
        self.value_dim = L['mask_decoder.gru'].weight.shape[0] // 3

    @staticmethod
    def _fusion(L, sd, p, n_shared):
        c1 = _fold(sd, p + '.block1.conv1', None, 1, 1)
        ds = _fold(sd, p + '.block1.downsample', None, 1, 0)
        L[p + '.b1.c1_x'], L[p + '.b1.c1_g'] = _split_in(c1, n_shared)
        L[p + '.b1.ds_x'], L[p + '.b1.ds_g'] = _split_in(ds, n_shared)
        L[p + '.b1.c2'] = _fold(sd, p + '.block1.conv2', None, 1, 1)
        L[p + '.b2.c1'] = _fold(sd, p + '.block2.conv1', None, 1, 1)
        L[p + '.b2.c2'] = _fold(sd, p + '.block2.conv2', None, 1, 1)


class TorchOps:
    """Interim backend: ATen/cuDNN ops on the device, fp32 NCHW (see module docstring)."""
    @staticmethod
    def conv(x, spec: ConvSpec, relu_in=False, relu_out=False, add=None):
        if relu_in:
            x = F.relu(x)
        y = F.conv2d(x, spec.weight, spec.bias, stride=spec.stride, padding=spec.pad)
        if add is not None:
            y = y + add
        return F.relu(y) if relu_out else y

    @staticmethod
    def maxpool(x):
        return F.max_pool2d(x, 3, 2, 1)

    @staticmethod
    def up2(x):
        return F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False)

    @staticmethod
    def area(x, ratio):
        return F.interpolate(x, scale_factor=ratio, mode='area')


class Engine:
    """Forward graphs.  Tensors between stages are NCHW fp32 on the device."""
    def __init__(self, sd: Dict[str, torch.Tensor]):
        self.t = LayerTable(sd)
        self.ops = TorchOps
        self.device = next(iter(sd.values())).device

    # ------------------------------------------------------------------ key encoder (a10, a11)
    def _bottleneck(self, x, q):
        L, ops = self.t.layers, self.ops
        y = ops.conv(x, L[q + '.c1'], relu_out=True)
        y = ops.conv(y, L[q + '.c2'], relu_out=True)
        short = ops.conv(x, L[q + '.ds']) if (q + '.ds') in L else x
        return ops.conv(y, L[q + '.c3'], add=short, relu_out=True)

    def encode_image(self, image):
        L, ops = self.t.layers, self.ops
        p = 'pixel_encoder'
        x = ops.maxpool(ops.conv(image, L[p + '.stem'], relu_out=True))
        feats = []
        for stage, blocks in (('res2', 3), ('layer2', 4), ('layer3', 6)):
            for i in range(blocks):
                x = self._bottleneck(x, f'{p}.{stage}.{i}')
            feats.append(x)
        f4, f8, f16 = feats
        return (ops.conv(f16, L[p + '.proj1']), f8, f4), ops.conv(f16, L[p + '.proj2'])

    def transform_key(self, feat, need_sk=True, need_ek=True):
        y = self.ops.conv(feat, self.t.layers['key_proj.all'])
        ck = self.t.key_dim
        key = y[:, :ck]
        shrinkage = y[:, ck:ck + 1]**2 + 1 if need_sk else None
        selection = torch.sigmoid(y[:, ck + 1:]) if need_ek else None
        return key, shrinkage, selection

    # ------------------------------------------------------------------ shared blocks
    def _cbam(self, x, p):
        c = self.t.cbam[p]

        def mlp(v):
            return F.linear(F.relu(F.linear(v, c['w1'], c['b1'])), c['w2'], c['b2'])

        gate = torch.sigmoid(mlp(x.mean((2, 3))) + mlp(x.amax((2, 3))))
        x = x * gate[:, :, None, None]
        pooled = torch.cat([x.amax(1, keepdim=True), x.mean(1, keepdim=True)], 1)
        return x * torch.sigmoid(F.conv2d(pooled, c['ws'], c['bs'], padding=3))

    def _fuse(self, p, x_shared, g):
        """GroupFeatureFusionBlock (group_modules.py:133-152) with the shared half hoisted out of the objects."""
        L, ops = self.t.layers, self.ops
        sx = ops.conv(x_shared, L[p + '.b1.c1_x'], relu_in=True)  # [1,mid,h,w], carries conv1's bias
        dx = ops.conv(x_shared, L[p + '.b1.ds_x'])  # carries downsample's bias
        y = ops.conv(g, L[p + '.b1.c1_g'], relu_in=True, add=sx)
        short = ops.conv(g, L[p + '.b1.ds_g'], add=dx)
        g = ops.conv(y, L[p + '.b1.c2'], relu_in=True, add=short)
        g = g + self._cbam(g, p)
        y = ops.conv(g, L[p + '.b2.c1'], relu_in=True)
        return ops.conv(y, L[p + '.b2.c2'], relu_in=True, add=g)

    @staticmethod
    def _gru(values, h):
        """Non-standard GRU of the reference (modules.py:145-149, quirk Q7)."""
        d = h.shape[1]
        f = torch.sigmoid(values[:, :d])
        u = torch.sigmoid(values[:, d:2 * d])
        return f * h * (1 - u) + u * torch.tanh(values[:, 2 * d:])

    def _resblock(self, q, g):
        L, ops = self.t.layers, self.ops
        y = ops.conv(g, L[q + '.c1'], relu_in=True)
        short = ops.conv(g, L[q + '.ds']) if (q + '.ds') in L else g
        return ops.conv(y, L[q + '.c2'], relu_in=True, add=short)

    # ------------------------------------------------------------------ value encoder (a13)
    def _basic(self, x, q):
        L, ops = self.t.layers, self.ops
        y = ops.conv(x, L[q + '.c1'], relu_out=True)
        short = ops.conv(x, L[q + '.ds']) if (q + '.ds') in L else x
        return ops.conv(y, L[q + '.c2'], add=short, relu_out=True)

    def encode_mask(self, image, ms_features, sensory, masks, deep_update=True, chunk_size=-1):
        """image [1,3,H,W], sensory [1,K,C,h,w], masks [1,K,H,W] -> (value [1,K,C,h,w], sensory')."""
        L, ops = self.t.layers, self.ops
        p = 'mask_encoder'
        k = masks.shape[1]
        step = k if chunk_size < 1 or chunk_size >= k else chunk_size
        stem_img = ops.conv(image, L[p + '.stem_img'])  # shared half of the 7x7 stem, once per frame
        new_sensory = sensory if (step == k or not deep_update) else torch.empty_like(sensory)
        values = []
        for i in range(0, k, step):
            m = masks[0, i:i + step].unsqueeze(1).float()
            x = ops.conv(m, L[p + '.stem_mask'], add=stem_img)
            x = F.relu(ops.maxpool(x))  # conv -> BN -> maxpool -> ReLU (quirk Q6)
            for stage in ('layer1', 'layer2', 'layer3'):
                for b in range(2):
                    x = self._basic(x, f'{p}.{stage}.{b}')
            g16 = self._fuse(p + '.fuser', ms_features[0], x)
            values.append(g16)
            if deep_update:
                h = sensory[0, i:i + step]
                nh = self._gru(ops.conv(torch.cat([g16, h], 1), L[p + '.gru']), h)
                if step == k:
                    new_sensory = nh.unsqueeze(0)
                else:
                    new_sensory[0, i:i + step] = nh
        value = values[0] if len(values) == 1 else torch.cat(values, 0)
        return value.unsqueeze(0), new_sensory

    # ------------------------------------------------------------------ decoder (a12, a14)
    @staticmethod
    def aggregate(prob, dim):
        """Soft aggregation (network.py:33-40), always fp32."""
        prob = prob.float()
        full = torch.cat([torch.prod(1 - prob, dim=dim, keepdim=True), prob], dim).clamp(1e-7, 1 - 1e-7)
        return torch.log(full / (1 - full))

    def decode(self, ms_features, readout, sensory, last_mask, update_sensory=True, chunk_size=-1):
        """readout/sensory [1,K,C,h,w], last_mask [1,K,H,W] -> (sensory', logits [1,K,H/4,W/4])."""
        L, ops = self.t.layers, self.ops
        p = 'mask_decoder'
        f16, f8, f4 = ms_features
        k = readout.shape[1]
        step = k if chunk_size < 1 or chunk_size >= k else chunk_size
        last = F.interpolate(last_mask.float(), size=readout.shape[-2:], mode='area')[0].unsqueeze(1)  # [K,1,h,w]
        skip8 = ops.conv(f8, L[p + '.skip8'])
        skip4 = ops.conv(f4, L[p + '.skip4'])
        new_sensory = sensory if (step == k or not update_sensory) else torch.empty_like(sensory)
        logits_all = []
        for i in range(0, k, step):
            h = sensory[0, i:i + step]
            p16 = ops.conv(torch.cat([h, last[i:i + step]], 1), L[p + '.sensory_compress'], add=readout[0, i:i + step])
            p16 = self._fuse(p + '.fuser', f16, p16)
            p8 = self._resblock(p + '.up_16_8.out_conv', ops.up2(p16) + skip8)
            p4 = self._resblock(p + '.up_8_4.out_conv', ops.up2(p8) + skip4)
            logits = ops.conv(p4, L[p + '.pred'], relu_in=True)  # [k,1,H/4,W/4]
            if update_sensory:
                g = ops.conv(p16, L[p + '.su.g16_conv']) + ops.conv(ops.area(p8, 1 / 2), L[p + '.su.g8_conv']) + \
                    ops.conv(ops.area(torch.cat([p4, logits], 1), 1 / 4), L[p + '.su.g4_conv'])
                nh = self._gru(ops.conv(torch.cat([g, h], 1), L[p + '.gru']), h)
                if step == k:
                    new_sensory = nh.unsqueeze(0)
                else:
                    new_sensory[0, i:i + step] = nh
            logits_all.append(logits)
        logits = logits_all[0] if len(logits_all) == 1 else torch.cat(logits_all, 0)
        return new_sensory, logits.view(1, k, *logits.shape[-2:])
