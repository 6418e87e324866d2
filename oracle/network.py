"""Oracle: DEVA propagation network as flat fp32 functions over a checkpoint state_dict.

Test infrastructure (see oracle/__init__.py).  Restates, layer for layer,
deva/model/network.py:33-173, big_modules.py:23-212, modules.py:22-169,
group_modules.py:17-152, cbam.py:21-77 and resnet.py:46-152 of the reference.  Nothing is
folded or reordered: BatchNorm stays a separate eval-mode op so the result is the
reference's fp32 arithmetic.  Every function keeps the dtype it is given, so a state dict and inputs upcast to float64
replay the same network in float64 (tests/test_engine_float64_gpu.py measures the native engine against that).

Tensor conventions follow the reference: images [1,3,H,W]; per-object tensors
[1,K,C,h,w]; ``sd`` is the flat checkpoint dict (``pixel_encoder.*``, ``mask_encoder.*``,
``key_proj.*``, ``mask_decoder.*``).
"""
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]


def _conv(sd: SD, name: str, x, stride=1, pad=0):
    return F.conv2d(x, sd[name + '.weight'], sd.get(name + '.bias'), stride=stride, padding=pad)


def _bn(sd: SD, name: str, x):
    return F.batch_norm(x, sd[name + '.running_mean'], sd[name + '.running_var'],
                        sd[name + '.weight'], sd[name + '.bias'], False, 0.0, 1e-5)


def _gconv(sd: SD, name: str, g, pad=0):
    """Per-object conv: objects ride in the batch dim.  group_modules.py:41-45."""
    b, k = g.shape[:2]
    y = _conv(sd, name, g.flatten(0, 1), pad=pad)
    return y.view(b, k, *y.shape[1:])


# ---------------------------------------------------------------------------- ResNet pieces
def _bottleneck(sd: SD, p: str, x, stride: int):
    """resnet.py:78-114."""
    y = F.relu(_bn(sd, p + '.bn1', _conv(sd, p + '.conv1', x)))
    y = F.relu(_bn(sd, p + '.bn2', _conv(sd, p + '.conv2', y, stride=stride, pad=1)))
    y = _bn(sd, p + '.bn3', _conv(sd, p + '.conv3', y))
    if (p + '.downsample.0.weight') in sd:
        x = _bn(sd, p + '.downsample.1', _conv(sd, p + '.downsample.0', x, stride=stride))
    return F.relu(y + x)


def _basic_block(sd: SD, p: str, x, stride: int):
    """resnet.py:46-75."""
    y = F.relu(_bn(sd, p + '.bn1', _conv(sd, p + '.conv1', x, stride=stride, pad=1)))
    y = _bn(sd, p + '.bn2', _conv(sd, p + '.conv2', y, pad=1))
    if (p + '.downsample.0.weight') in sd:
        x = _bn(sd, p + '.downsample.1', _conv(sd, p + '.downsample.0', x, stride=stride))
    return F.relu(y + x)


def _stage(sd: SD, p: str, x, blocks: int, stride: int, block_fn):
    for i in range(blocks):
        x = block_fn(sd, f'{p}.{i}', x, stride if i == 0 else 1)
    return x


# ------------------------------------------------------------------------------ key encoder
def encode_image(sd: SD, image):
    """network.py:42-44 -> big_modules.py:42-51.  Returns ((f16, f8, f4), key_feat)."""
    p = 'pixel_encoder'
    x = F.relu(_bn(sd, p + '.bn1', _conv(sd, p + '.conv1', image, stride=2, pad=3)))
    x = F.max_pool2d(x, 3, 2, 1)
    f4 = _stage(sd, p + '.res2', x, 3, 1, _bottleneck)
    f8 = _stage(sd, p + '.layer2', f4, 4, 2, _bottleneck)
    f16 = _stage(sd, p + '.layer3', f8, 6, 2, _bottleneck)
    return (_conv(sd, p + '.proj1', f16), f8, f4), _conv(sd, p + '.proj2', f16)


def transform_key(sd: SD, feat):
    """network.py:62-68 -> modules.py:73-78.  Returns (key, shrinkage, selection)."""
    shrinkage = _conv(sd, 'key_proj.d_proj', feat, pad=1)**2 + 1
    selection = torch.sigmoid(_conv(sd, 'key_proj.e_proj', feat, pad=1))
    return _conv(sd, 'key_proj.key_proj', feat, pad=1), shrinkage, selection


# ----------------------------------------------------------------------------- shared blocks
def _group_resblock(sd: SD, p: str, g):
    """group_modules.py:48-67."""
    y = _gconv(sd, p + '.conv1', F.relu(g), pad=1)
    y = _gconv(sd, p + '.conv2', F.relu(y), pad=1)
    if (p + '.downsample.weight') in sd:
        g = _gconv(sd, p + '.downsample', g)
    return y + g


def _cbam(sd: SD, p: str, x):
    """cbam.py:21-77 on [B,C,h,w]."""
    def mlp(v):
        v = F.relu(F.linear(v, sd[p + '.ChannelGate.mlp.1.weight'], sd[p + '.ChannelGate.mlp.1.bias']))
        return F.linear(v, sd[p + '.ChannelGate.mlp.3.weight'], sd[p + '.ChannelGate.mlp.3.bias'])

    att = mlp(x.mean((2, 3))) + mlp(x.amax((2, 3)))
    x = x * torch.sigmoid(att)[:, :, None, None]
    pooled = torch.cat([x.amax(1, keepdim=True), x.mean(1, keepdim=True)], 1)
    gate = torch.sigmoid(_conv(sd, p + '.SpatialGate.spatial.conv', pooled, pad=3))
    return x * gate


def _fusion(sd: SD, p: str, x, g):
    """group_modules.py:133-152: cat[x broadcast, g] -> ResBlock -> +CBAM -> ResBlock."""
    b, k = g.shape[:2]
    g = torch.cat([x.unsqueeze(1).expand(-1, k, -1, -1, -1), g], 2)
    g = _group_resblock(sd, p + '.block1', g)
    r = _cbam(sd, p + '.attention', g.flatten(0, 1)).view_as(g)
    return _group_resblock(sd, p + '.block2', g + r)


def _gru(values, h, dim: int):
    """modules.py:145-149 / :163-167 (the non-standard gate order, quirk Q7)."""
    f = torch.sigmoid(values[:, :, :dim])
    u = torch.sigmoid(values[:, :, dim:2 * dim])
    n = torch.tanh(values[:, :, 2 * dim:])
    return f * h * (1 - u) + u * n


def _resize_groups(g, ratio, mode):
    b, k = g.shape[:2]
    kw = dict(align_corners=False) if mode == 'bilinear' else {}
    y = F.interpolate(g.flatten(0, 1), scale_factor=ratio, mode=mode, **kw)
    return y.view(b, k, *y.shape[1:])


# ---------------------------------------------------------------------------- value encoder
def encode_mask(sd: SD, image, ms_features, sensory, masks, deep_update=True):
    """network.py:46-60 -> big_modules.py:73-127.  masks [1,K,H,W] -> (value, new_sensory)."""
    p = 'mask_encoder'
    b, k = masks.shape[:2]
    g = torch.cat([image.unsqueeze(1).expand(-1, k, -1, -1, -1), masks.unsqueeze(2)], 2)
    x = g.flatten(0, 1)
    x = _bn(sd, p + '.bn1', _conv(sd, p + '.conv1', x, stride=2, pad=3))
    x = F.relu(F.max_pool2d(x, 3, 2, 1))  # conv -> BN -> maxpool -> ReLU (quirk Q6)
    x = _stage(sd, p + '.layer1', x, 2, 1, _basic_block)
    x = _stage(sd, p + '.layer2', x, 2, 2, _basic_block)
    x = _stage(sd, p + '.layer3', x, 2, 2, _basic_block)
    g16 = _fusion(sd, p + '.fuser', ms_features[0], x.view(b, k, *x.shape[1:]))
    if deep_update:
        vals = _gconv(sd, p + '.sensory_update.transform', torch.cat([g16, sensory], 2), pad=1)
        sensory = _gru(vals, sensory, sensory.shape[2])
    return g16, sensory


# ---------------------------------------------------------------------------------- decoder
def _at_least_f32(x):
    """The reference's ``.float()``, except that float64 stays float64 (a float64 replay of the network)."""
    return x.to(torch.promote_types(x.dtype, torch.float32))


def aggregate(prob, dim: int):
    """network.py:33-40."""
    prob = _at_least_f32(prob)
    full = torch.cat([torch.prod(1 - prob, dim=dim, keepdim=True), prob], dim).clamp(1e-7, 1 - 1e-7)
    return torch.log(full / (1 - full))


def segment(sd: SD, ms_features, readout, sensory, last_mask, update_sensory=True):
    """network.py:94-173 (inference branch) -> big_modules.py:147-212.

    readout/sensory [1,K,512,h,w]; last_mask [1,K,H,W].  Returns (sensory, logits, prob).
    """
    sensory, logits = decode(sd, ms_features, readout, sensory, last_mask, update_sensory)
    logits, prob = output_tail(logits)
    return sensory, logits, prob


def decode(sd: SD, ms_features, readout, sensory, last_mask, update_sensory=True):
    """The decoder up to the logits, before the objects meet in ``aggregate``: every object's result depends on its own
    readout / sensory / mask only (quirk Q11), so the objects can be run one at a time.

    readout/sensory [1,K,512,h,w]; last_mask [1,K,H,W].  Returns (sensory, logits [1,K,H/4,W/4]).
    """
    p = 'mask_decoder'
    f16, f8, f4 = ms_features
    b, k = readout.shape[:2]
    last = F.interpolate(last_mask, size=readout.shape[-2:], mode='area').unsqueeze(2)
    skip8 = _conv(sd, p + '.decoder_feat_proc.transforms.0', f8)
    skip4 = _conv(sd, p + '.decoder_feat_proc.transforms.1', f4)

    p16 = readout + _gconv(sd, p + '.sensory_compress', torch.cat([sensory, last], 2))
    p16 = _fusion(sd, p + '.fuser', f16, p16)
    p8 = _group_resblock(sd, p + '.up_16_8.out_conv', skip8.unsqueeze(1) + _resize_groups(p16, 2, 'bilinear'))
    p4 = _group_resblock(sd, p + '.up_8_4.out_conv', skip4.unsqueeze(1) + _resize_groups(p8, 2, 'bilinear'))
    logits = _conv(sd, p + '.pred', F.relu(_at_least_f32(p4.flatten(0, 1))), pad=1)

    if update_sensory:
        p4x = torch.cat([p4, logits.view(b, k, 1, *logits.shape[-2:])], 2)
        su = p + '.sensory_update'
        g = _gconv(sd, su + '.g16_conv', p16) + \
            _gconv(sd, su + '.g8_conv', _resize_groups(p8, 1 / 2, 'area')) + \
            _gconv(sd, su + '.g4_conv', _resize_groups(p4x, 1 / 4, 'area'))
        vals = _gconv(sd, su + '.transform', torch.cat([g, sensory], 2), pad=1)
        sensory = _gru(vals, sensory, sensory.shape[2])
    return sensory, logits.view(b, k, *logits.shape[-2:])


def output_tail(logits):
    """network.py:144 and :164-168: per-object logits [1,K,h4,w4] -> soft aggregation over all K objects, x4 bilinear,
    softmax.  Returns (aggregated logits [1,K+1,4*h4,4*w4], prob)."""
    prob = torch.sigmoid(logits)
    logits = aggregate(prob, dim=1)
    logits = F.interpolate(logits, scale_factor=4, mode='bilinear', align_corners=False)
    return logits, F.softmax(logits, dim=1)
