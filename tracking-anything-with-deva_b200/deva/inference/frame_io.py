"""Frame ingest / egress around ``DEVAInferenceCore.step`` (SURVEY 8f-3): the two per-frame host<->device hops of a
real pipeline, each as one kernel.

* ``frame_from_rgb8``: the decoded uint8 frame is uploaded as is (3 bytes / pixel instead of 12) and ToTensor +
  Normalize (deva/inference/data/video_reader.py:146-150, IMAGENET mean/std) run on the device - bit-exact.  With
  ``size`` it also resizes to the working resolution the way the reference's drivers do, on the device: the readers'
  ``Resize(size, BILINEAR, antialias=True)`` (video_reader.py:151, detection_video_reader.py:67-70) or demo_utils'
  plain bilinear ``F.interpolate`` (demo_utils.py:10-19), optionally followed by eval_vos.py:162-164's flip.
* ``mask_from_index8``: the first-frame / detection index mask through the readers' ``Resize(size, NEAREST)`` (PIL's
  nearest, not torch's) and the same optional flip.
* ``prob_to_ids``: the driver's post-step (evaluation/eval_vos.py:169-181) - bilinear resize to the original size,
  optional flip, argmax, ``ObjectManager.tmp_to_obj_cls`` - fused into a single pass that writes the id map.
* ``prob_to_segments``: the same resize and argmax plus everything the result savers derive from the id map (index
  mask, long-id RGB image, visualisation overlay, per-segment areas and boxes), in one pass.
* ``prob_to_scores`` / ``scores_to_ids``: multi-scale / flip evaluation - eval_vos.py's ``--save_scores`` array (the
  same resize and flip, quantised to uint8) and scripts/merge_multi_scale.py's merge of the members' arrays (sum,
  argmax, ``{object id: tmp id}`` remap).
"""
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from deva import _native as nat

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def reader_size(h: int, w: int, size: int) -> Tuple[int, int]:
    """Output (h, w) of torchvision's ``Resize(size)`` (the readers' convention): short side = size, long side =
    int(size * long / short)."""
    short, long = (w, h) if w <= h else (h, w)
    new_short, new_long = size, int(size * long / short)
    return (new_long, new_short) if w <= h else (new_short, new_long)


def demo_size(h: int, w: int, size: int) -> Tuple[int, int]:
    """Output (h, w) of demo_utils.get_input_frame_for_deva: scale = size / min(h, w), (int(h * scale), int(w * scale))."""
    scale = size / min(h, w)
    return int(h * scale), int(w * scale)


def antialias_taps(n_in: int, n_out: int) -> Tuple[np.ndarray, np.ndarray]:
    """int32 / float32 [n_out, taps] source indices and weights of torch's CPU ``_upsample_bilinear2d_aa`` along one
    axis (align_corners=False): a triangle filter whose support is scaled by the downscale factor, weights normalised
    per output pixel.  Float32 where torch's kernel keeps float, double where its expressions promote to double.
    Unused taps have weight 0 and repeat the last index."""
    f32, f64 = np.float32, np.float64
    scale = f32(n_in) / f32(n_out)
    support = scale if scale >= 1 else f32(1.0)
    taps = int(np.ceil(support)) * 2 + 1
    invscale = f32(1.0 / f64(scale)) if scale >= 1 else f32(1.0)
    center = (f64(scale) * (np.arange(n_out, dtype=f64) + 0.5)).astype(f32)
    xmin = np.maximum((f64(center - support) + 0.5).astype(np.int64), 0)
    xsize = np.clip(np.minimum((f64(center + support) + 0.5).astype(np.int64), n_in) - xmin, 0, taps)
    j = np.arange(taps)
    x = np.abs(((f64((xmin[:, None] + j).astype(f32) - center[:, None]) + 0.5) * f64(invscale)).astype(f32))
    wt = np.where(x < 1, f32(1) - x, f32(0)).astype(f32)
    wt[j >= xsize[:, None]] = 0
    total = np.zeros(n_out, f32)
    for k in range(taps):  # torch sums the weights in tap order
        total = total + wt[:, k]
    wt = np.where(total[:, None] != 0, wt / np.where(total == 0, f32(1), total)[:, None], wt).astype(f32)
    idx = np.minimum(xmin[:, None] + np.minimum(j, np.maximum(xsize[:, None] - 1, 0)), n_in - 1)
    return idx.astype(np.int32), wt


def bilinear_taps(n_in: int, n_out: int) -> Tuple[np.ndarray, np.ndarray]:
    """int32 / float32 [n_out, 2] source indices and weights of torch's CPU ``upsample_bilinear2d``
    (align_corners=False) along one axis.  The source coordinate scale * (o + 0.5) - 0.5 is one fused multiply-add in
    float32, as torch's kernel computes it."""
    f32, f64 = np.float32, np.float64
    scale = f32(n_in) / f32(n_out)
    real = np.maximum((f64(scale) * (np.arange(n_out) + 0.5) - 0.5).astype(f32), f32(0))
    i0 = np.minimum(np.floor(real).astype(np.int64), n_in - 1)
    lam = np.clip(real - i0.astype(f32), f32(0), f32(1)).astype(f32)
    i1 = i0 + (i0 < n_in - 1)
    return np.stack([i0, i1], 1).astype(np.int32), np.stack([f32(1) - lam, lam], 1)


def pil_nearest_map(n_in: int, n_out: int) -> np.ndarray:
    """int32 [n_out] source index of PIL's NEAREST resize along one axis: PIL steps a double coordinate from
    0.5 * n_in / n_out by n_in / n_out and truncates it (ImagingScaleAffine), which is not torch's 'nearest'."""
    a = n_in / n_out
    out, xo = np.empty(n_out, np.int32), a * 0.5
    for o in range(n_out):
        out[o] = min(int(xo), n_in - 1)
        xo += a
    return out


def pil_bilinear_coeffs(n_in: int, n_out: int) -> Tuple[np.ndarray, np.ndarray]:
    """int32 [n_out, 2] (first input index, taps) and int32 [n_out, taps] 22-bit fixed-point coefficients of Pillow's
    8-bit BILINEAR resample along one axis (libImaging Resample.c: precompute_coeffs, then normalize_coeffs_8bpc): a
    triangle whose support is scaled by the downscale factor, double arithmetic, weights normalised per output pixel
    and rounded half away from zero.  Unused taps are 0."""
    scale = float(np.float32(n_in)) / n_out
    filterscale = max(scale, 1.0)
    support = filterscale
    taps = int(np.ceil(support)) * 2 + 1
    center = (np.arange(n_out, dtype=np.float64) + 0.5) * scale
    lo = np.maximum((center - support + 0.5).astype(np.int64), 0)
    n = np.minimum((center + support + 0.5).astype(np.int64), n_in) - lo
    x = np.abs(((lo[:, None] + np.arange(taps)).astype(np.float64) - center[:, None] + 0.5) * (1.0 / filterscale))
    wt = np.where(x < 1.0, 1.0 - x, 0.0)
    wt[np.arange(taps)[None, :] >= n[:, None]] = 0.0
    total = np.zeros(n_out)
    for j in range(taps):  # Pillow sums the weights in tap order
        total = total + wt[:, j]
    wt = np.where(total[:, None] != 0.0, wt / np.where(total == 0.0, 1.0, total)[:, None], wt)
    fixed = np.trunc(wt * (1 << 22) + np.where(wt < 0, -0.5, 0.5)).astype(np.int32)
    return np.stack([lo, n], 1).astype(np.int32), fixed


_TABLES: Dict[tuple, Tuple[torch.Tensor, ...]] = {}


def _axis_table(kind: str, n_in: int, n_out: int, device) -> Tuple[torch.Tensor, ...]:
    """Device copy of one axis' resampling table, built on the host once per (kind, n_in, n_out, device)."""
    key = (kind, n_in, n_out, torch.device(device))
    if key not in _TABLES:
        if kind == 'nearest':
            arrays = (pil_nearest_map(n_in, n_out),)
        elif kind == 'pil_bilinear':
            arrays = pil_bilinear_coeffs(n_in, n_out)
        else:
            arrays = (antialias_taps if kind == 'antialias' else bilinear_taps)(n_in, n_out)
        _TABLES[key] = tuple(torch.from_numpy(a).to(device) for a in arrays)
    return _TABLES[key]


def _to_device(t: torch.Tensor, device) -> torch.Tensor:
    if not t.is_cuda:
        t = t.to(device or torch.device('cuda', torch.cuda.current_device()), non_blocking=True)
    return t.contiguous()


def frame_from_rgb8(frame: torch.Tensor, mean: Sequence[float] = IMAGENET_MEAN, std: Sequence[float] = IMAGENET_STD,
                    device: Optional[torch.device] = None, *, size: Optional[int] = None, resize: str = 'reader',
                    flip: bool = False) -> torch.Tensor:
    """uint8 [H, W, 3] RGB (host - ideally pinned - or device) -> normalised float32 [3, H', W'] on the device.

    ``size`` (None: keep H, W) is the working resolution's short side.  ``resize='reader'`` sizes the output like
    torchvision's ``Resize(size)`` and filters like the readers (antialiased bilinear); ``resize='demo'`` sizes and
    filters like demo_utils (plain bilinear).  ``flip`` mirrors the resized frame horizontally.  An output the size of
    the input is the plain normalised frame, bit for bit, as the reference's resize returns its input unchanged."""
    assert frame.dtype == torch.uint8 and frame.dim() == 3 and frame.shape[2] == 3
    assert resize in ('reader', 'demo'), resize
    assert size is None or size > 0, size
    frame = _to_device(frame, device)
    h, w = frame.shape[:2]
    oh, ow = (h, w) if size is None else (reader_size if resize == 'reader' else demo_size)(h, w, size)
    out = torch.empty(3, oh, ow, dtype=torch.float32, device=frame.device)
    if (oh, ow) == (h, w) and not flip:
        nat.ingest_rgb8(frame, out, h, w, mean, std)
        return out
    kind = 'antialias' if resize == 'reader' else 'bilinear'
    x_idx, x_w = _axis_table(kind, w, ow, frame.device)
    y_idx, y_w = _axis_table(kind, h, oh, frame.device)
    scratch = torch.empty(3, h, ow, dtype=torch.float32, device=frame.device)
    nat.ingest_rgb8_resize(frame, h, w, oh, ow, x_idx, x_w, y_idx, y_w, scratch, out, flip, mean, std)
    return out


def mask_from_index8(mask: torch.Tensor, size: Optional[int] = None, *, flip: bool = False,
                     device: Optional[torch.device] = None) -> torch.Tensor:
    """uint8 [H, W] index mask (host or device) -> int64 [H', W'] on the device: the readers' ``Resize(size, NEAREST)``
    on the PIL mask (output size as torchvision's ``Resize(size)``), then an optional horizontal flip."""
    assert mask.dtype == torch.uint8 and mask.dim() == 2
    assert size is None or size > 0, size
    mask = _to_device(mask, device)
    h, w = mask.shape
    oh, ow = (h, w) if size is None else reader_size(h, w, size)
    (x_idx,), (y_idx,) = _axis_table('nearest', w, ow, mask.device), _axis_table('nearest', h, oh, mask.device)
    out = torch.empty(oh, ow, dtype=torch.long, device=mask.device)
    nat.mask_nearest(mask, h, w, oh, ow, x_idx, y_idx, flip, out)
    return out


def mask_ids_from_u8(mask: torch.Tensor, size: Optional[int] = None, *, device: Optional[torch.device] = None,
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """uint8 [H, W] index mask or [H, W, 3] RGB mask (host or device) -> int32 [H', W'] ids on the device: the
    detection reader's ``Resize(size, NEAREST)`` (PIL's nearest, output size as torchvision's ``Resize(size)``), then
    the index itself, or ``r + 256 g + 65536 b`` for RGB.  ``out`` (int32 [H', W'] on the device) receives the ids."""
    assert mask.dtype == torch.uint8 and (mask.dim() == 2 or (mask.dim() == 3 and mask.shape[2] == 3)), mask.shape
    assert size is None or size > 0, size
    mask = _to_device(mask, device)
    h, w = mask.shape[:2]
    oh, ow = (h, w) if size is None else reader_size(h, w, size)
    (x_idx,), (y_idx,) = _axis_table('nearest', w, ow, mask.device), _axis_table('nearest', h, oh, mask.device)
    if out is None:
        out = torch.empty(oh, ow, dtype=torch.int32, device=mask.device)
    assert out.dtype == torch.int32 and out.is_contiguous() and tuple(out.shape) == (oh, ow), (out.dtype, out.shape)
    nat.mask_nearest_ids(mask, 1 if mask.dim() == 2 else 3, h, w, oh, ow, x_idx, y_idx, False, out)
    return out


def soft_from_u8(planes: torch.Tensor, size: Optional[int] = None, *, device: Optional[torch.device] = None,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """uint8 [K, H, W] soft-mask planes (host or device) -> float32 [K, H', W'] on the device: per plane the reader's
    ``Resize(size, BILINEAR)`` of an L image (Pillow's 8-bit resample, bit for bit; output size as torchvision's
    ``Resize(size)``), then ``torch.FloatTensor(np.array(mask)) / 255``.  One launch per pass for all K planes."""
    assert planes.dtype == torch.uint8 and planes.dim() == 3 and planes.shape[0] > 0, (planes.dtype, planes.shape)
    assert size is None or size > 0, size
    planes = _to_device(planes, device)
    k, h, w = planes.shape
    oh, ow = (h, w) if size is None else reader_size(h, w, size)
    if out is None:
        out = torch.empty(k, oh, ow, dtype=torch.float32, device=planes.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (k, oh, ow), (out.dtype, out.shape)
    xb, xc = _axis_table('pil_bilinear', w, ow, planes.device) if ow != w else (None, None)
    yb, yc = _axis_table('pil_bilinear', h, oh, planes.device) if oh != h else (None, None)
    scratch = torch.empty(k, h, ow, dtype=torch.uint8, device=planes.device) if ow != w and oh != h else None
    nat.pil_resample_u8(planes, k, h, w, oh, ow, xb, xc, yb, yc, scratch, out)
    return out


def _lut_list(object_manager, channels: int) -> List[int]:
    lut = [0] * channels
    for tmp_id, obj in object_manager.tmp_id_to_obj.items():
        if 0 < tmp_id < channels:
            lut[tmp_id] = int(obj.id)
    return lut


def id_lut(object_manager, channels: int, device) -> torch.Tensor:
    """int32 [channels]: temporary id (prob channel) -> object id; channel 0 and unknown channels -> 0."""
    return torch.tensor(_lut_list(object_manager, channels), dtype=torch.int32, device=device)


def id_rgb(i: int) -> int:
    """ID2RGBConverter._id_to_rgb(i) (deva/utils/pano_utils.py) packed as r | g << 8 | b << 16: the bytes i % 256,
    i // 256 % 256, i // 65536 % 256."""
    return (i % 256) | (i // 256 % 256) << 8 | (i // 65536 % 256) << 16


def segment_tables(object_manager, channels: int, remap: bool = True) -> Tuple[List[int], List[int]]:
    """Host tables of ``prob_to_segments``: ``lut`` [channels], the value written for each channel (its object id,
    or the channel itself when ``remap`` is False), and ``rgb`` [channels], the packed colour of that value when it
    is the id of a current object, else 0 (the saver colours only ``all_obj_ids``, result_utils.py:208-215)."""
    lut = _lut_list(object_manager, channels) if remap else list(range(channels))
    coloured = {int(o.id) for o in object_manager.obj_to_tmp_id}
    return lut, [id_rgb(v) if v in coloured else 0 for v in lut]


def prob_to_ids(prob: torch.Tensor, object_manager=None, size: Optional[Tuple[int, int]] = None, flip: bool = False,
                dtype: torch.dtype = torch.long, lut: Optional[torch.Tensor] = None) -> torch.Tensor:
    """prob float32 [K+1, H, W] from ``step`` -> id map [H0, W0] (``size`` or H, W), dtype long or uint8.

    Equals ``tmp_to_obj_cls(argmax(flip(interpolate(prob, size, 'bilinear', align_corners=False))))``."""
    assert prob.is_cuda and prob.dtype == torch.float32 and prob.dim() == 3 and dtype in (torch.long, torch.uint8)
    prob = prob.contiguous()
    c, h, w = prob.shape
    oh, ow = (h, w) if size is None else (int(size[0]), int(size[1]))
    if lut is None and object_manager is not None:
        lut = id_lut(object_manager, c, prob.device)
    out = torch.empty(oh, ow, dtype=dtype, device=prob.device)
    nat.prob_to_ids(prob, c, h, w, oh, ow, flip, lut, out if dtype == torch.uint8 else None,
                    out if dtype == torch.long else None)
    return out


@dataclass
class Segments:
    """Result of ``prob_to_segments``.  Device tensors, each None unless requested; ``lut`` is the host table the
    call used (channel -> value in ``index``), so per-channel ``counts`` / ``boxes`` can be grouped by id."""
    lut: List[int]
    index: Optional[torch.Tensor] = None  # uint8 [H0, W0]: (uint8) lut[argmax]
    rgb: Optional[torch.Tensor] = None  # uint8 [H0, W0, 3]: long-id colour image
    overlay: Optional[torch.Tensor] = None  # uint8 [H0, W0, 3]: frame blended with ``rgb``
    counts: Optional[torch.Tensor] = None  # int64 [K+1]: pixels per channel
    boxes: Optional[torch.Tensor] = None  # int32 [K+1, 4]: x_min, y_min, x_max, y_max per channel


def prob_to_segments(prob: torch.Tensor, object_manager, size: Optional[Tuple[int, int]] = None, *, index: bool = True,
                     rgb: bool = False, frame: Optional[torch.Tensor] = None, stats: bool = False,
                     remap: bool = True) -> Segments:
    """prob float32 [K+1, H, W] from ``step`` -> the result savers' per-frame outputs at ``size`` (or H, W), one pass.

    The argmax is ``prob_to_ids``' (its id map, bit for bit, without flip).  ``index``: the uint8 id mask (ids above
    255 wrap, like the saver's ``astype(np.uint8)``).  ``rgb``: the long-id RGB image.  ``frame`` (device uint8
    [H0, W0, 3]): the overlay, ``frame`` where the id is 0 and ``(frame + rgb) // 2`` elsewhere.  ``stats``: per-channel
    pixel counts and bounding boxes (empty channels: (INT32_MAX, INT32_MAX, -1, -1)).  ``remap`` False keeps the
    channel index instead of the object id.  Only enqueues work: no host synchronisation."""
    assert prob.is_cuda and prob.dtype == torch.float32 and prob.dim() == 3
    prob = prob.contiguous()
    c, h, w = prob.shape
    oh, ow = (h, w) if size is None else (int(size[0]), int(size[1]))
    dev = prob.device
    lut, colours = segment_tables(object_manager, c, remap)
    tables = torch.tensor([lut, colours], dtype=torch.int64).to(torch.int32).pin_memory().to(dev, non_blocking=True)
    if frame is not None:
        assert frame.is_cuda and frame.dtype == torch.uint8 and tuple(frame.shape) == (oh, ow, 3), frame.shape
        frame = frame.contiguous()
    out = Segments(lut)
    if index:
        out.index = torch.empty(oh, ow, dtype=torch.uint8, device=dev)
    if rgb:
        out.rgb = torch.empty(oh, ow, 3, dtype=torch.uint8, device=dev)
    if frame is not None:
        out.overlay = torch.empty(oh, ow, 3, dtype=torch.uint8, device=dev)
    if stats:
        out.counts = torch.empty(c, dtype=torch.int64, device=dev)
        out.boxes = torch.empty(c, 4, dtype=torch.int32, device=dev)
    nat.prob_to_segments(prob, c, h, w, oh, ow, tables[0], tables[1], frame, out.index, out.rgb, out.overlay,
                         out.counts, out.boxes)
    return out


def prob_to_scores(prob: torch.Tensor, size: Optional[Tuple[int, int]] = None, flip: bool = False, *,
                   scores: bool = True, into: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
    """prob float32 [K+1, H, W] from ``step`` -> uint8 scores [K+1, H0, W0] (``size`` or H, W) on the device.

    Equals ``(flip(interpolate(prob, size, 'bilinear', align_corners=False)) * 255).astype(np.uint8)``, the array
    eval_vos.py writes with ``--save_scores``: the resize and flip are ``prob_to_ids``' (the same values, bit for bit),
    the product one float32 multiply, truncated.  ``into`` (int32 [K+1, H0, W0] on the device) gets the scores added
    in the same pass: the running sum of a multi-scale / flip merge.  Returns the scores, or None with
    ``scores=False`` (then ``into`` is required).  Only enqueues work: no host synchronisation."""
    assert prob.is_cuda and prob.dtype == torch.float32 and prob.dim() == 3
    prob = prob.contiguous()
    c, h, w = prob.shape
    oh, ow = (h, w) if size is None else (int(size[0]), int(size[1]))
    if into is not None:
        if not (into.is_cuda and into.dtype == torch.int32 and into.is_contiguous() and into.device == prob.device):
            raise RuntimeError(f'prob_to_scores: into must be a contiguous int32 tensor on {prob.device}')
        if tuple(into.shape) != (c, oh, ow):
            raise RuntimeError(f'prob_to_scores: into has shape {tuple(into.shape)}, expected {(c, oh, ow)}')
    if not scores and into is None:
        raise RuntimeError('prob_to_scores: nothing to write (scores=False and no into)')
    out = torch.empty(c, oh, ow, dtype=torch.uint8, device=prob.device) if scores else None
    nat.prob_to_scores(prob, c, h, w, oh, ow, flip, out, into)
    return out


def mapping_lut(mapping: Dict[int, int], channels: int) -> List[int]:
    """``{object id: tmp id}`` (``ObjectManager.get_tmp_to_obj_mapping()``, eval_vos' backward.hkl) -> the value of
    each channel in merge_multi_scale.py's remap loop: ``idx_mask[argmax == tmp] = object id`` for every entry in
    order, so a later entry for the same channel overwrites an earlier one, and a channel no entry names stays 0."""
    lut = [0] * channels
    for obj_id, tmp in mapping.items():
        if 0 <= tmp < channels:
            lut[tmp] = int(obj_id)
    return lut


def scores_to_ids(total: torch.Tensor, object_manager=None, *, mapping: Optional[Dict[int, int]] = None,
                  dtype: torch.dtype = torch.uint8) -> torch.Tensor:
    """Summed scores int32 [K+1, H, W] -> id map [H, W] (uint8 or long) on the device: merge_multi_scale.py's
    ``np.argmax`` over channels (the first maximum wins a tie) and its remap through ``mapping`` (``{object id:
    tmp id}``; default ``object_manager.get_tmp_to_obj_mapping()``, with neither the channel itself).  uint8 ids
    above 255 wrap.  Only enqueues work: no host synchronisation."""
    assert dtype in (torch.long, torch.uint8), dtype
    if not (total.is_cuda and total.dtype == torch.int32 and total.dim() == 3):
        raise RuntimeError(f'scores_to_ids: expected int32 [K+1, H, W] on the device, got {total.dtype} '
                           f'{tuple(total.shape)} on {total.device}')
    total = total.contiguous()
    c, h, w = total.shape
    if mapping is None and object_manager is not None:
        mapping = object_manager.get_tmp_to_obj_mapping()
    lut = None
    if mapping is not None:
        lut = torch.tensor(mapping_lut(mapping, c), dtype=torch.int32).pin_memory().to(total.device, non_blocking=True)
    out = torch.empty(h, w, dtype=dtype, device=total.device)
    nat.scores_to_ids(total, c, h, w, lut, out if dtype == torch.uint8 else None, out if dtype == torch.long else None)
    return out
