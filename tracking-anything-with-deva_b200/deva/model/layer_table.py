"""The DEVA propagation network's convolutions as a flat, BN-folded layer table.

The reference builds the network as an ``nn.Module`` tree (deva/model/big_modules.py, modules.py,
group_modules.py, cbam.py, resnet.py).  ``LayerTable`` flattens it into one ``ConvSpec`` per convolution,
keyed by a dotted layer name, plus the fusers' CBAM weights; ``NativeEngine`` packs its kernel operands from
it.  Loading

* folds every eval-mode BatchNorm into the preceding bias-free convolution
  (w' = w * g/sqrt(var+eps), b' = beta - mean * g/sqrt(var+eps));
* splits convolutions whose input is ``cat[shared image feature, per-object feature]`` into a
  once-per-frame shared half and a per-object half (SURVEY.md section 7, hard part 5): the 7x7 stem of the
  mask encoder (image 3ch shared / mask 1ch per object) and ``fuser.block1.{conv1,downsample}`` of both
  fusers (512 shared / 256|512 per object);
* merges the three 3x3 key-projection heads, which share their input, into one convolution.
"""
from typing import Dict, Optional, Tuple

import torch

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
