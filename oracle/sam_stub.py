"""A stand-in ``segment_anything`` package and a fake SAM model, for running the reference's automatic mask generator
(deva/ext/SAM/automatic_mask_generator.py, unmodified) and this package's DeviceMaskGenerator without the real networks.

``segment_anything`` is not installed where this project is built, so the helper semantics below are RESTATED from
segment_anything's ``utils/amg.py`` (MaskData, batch_iterator, build_point_grid, calculate_stability_score,
batched_mask_to_box, crop boxes and uncropping), ``modeling/sam.py`` (Sam.postprocess_masks, mask_threshold),
``predictor.py`` (SamPredictor.set_image / predict_torch) and ``utils/transforms.py`` (ResizeLongestSide), without the
package.  tests/test_sam_masks_cpu.py compares them with the real package where it is installed.

``install()`` puts the modules into ``sys.modules`` (returning what it replaced, for ``uninstall``); the package never
imports this file.  ``FakeSam`` is a ``Sam`` whose image encoder does nothing and whose mask decoder returns seeded,
smooth low-resolution logits per prompt: a cone around the prompt with a per-mask radius and slope (so stability
scores straddle 0.95), predicted IoUs on a 1/32 grid (so they straddle 0.88 and tie), a few masks entirely below -1
(zero unions), and negative prompts carving holes.
"""
import math
import sys
import types
from copy import deepcopy
from typing import Any, Generator, List, Tuple

import numpy as np
import torch
import torch.nn.functional as F

# ---------------------------------------------------------------------------------------------- utils/amg.py


class MaskData:
    """A structure for storing masks and their related data in batched format."""

    def __init__(self, **kwargs) -> None:
        for v in kwargs.values():
            assert isinstance(v, (list, np.ndarray, torch.Tensor)), 'MaskData only supports list, numpy arrays, and torch tensors.'
        self._stats = dict(**kwargs)

    def __setitem__(self, key, item) -> None:
        assert isinstance(item, (list, np.ndarray, torch.Tensor)), 'MaskData only supports list, numpy arrays, and torch tensors.'
        self._stats[key] = item

    def __delitem__(self, key) -> None:
        del self._stats[key]

    def __getitem__(self, key):
        return self._stats[key]

    def items(self):
        return self._stats.items()

    def filter(self, keep: torch.Tensor) -> None:
        for k, v in self._stats.items():
            if v is None:
                self._stats[k] = None
            elif isinstance(v, torch.Tensor):
                self._stats[k] = v[torch.as_tensor(keep, device=v.device)]
            elif isinstance(v, np.ndarray):
                self._stats[k] = v[keep.detach().cpu().numpy()]
            elif isinstance(v, list) and keep.dtype == torch.bool:
                self._stats[k] = [a for i, a in enumerate(v) if keep[i]]
            elif isinstance(v, list):
                self._stats[k] = [v[i] for i in keep]
            else:
                raise TypeError(f'MaskData key {k} has an unsupported type {type(v)}.')

    def cat(self, new_stats: 'MaskData') -> None:
        for k, v in new_stats.items():
            if k not in self._stats or self._stats[k] is None:
                self._stats[k] = deepcopy(v)
            elif isinstance(v, torch.Tensor):
                self._stats[k] = torch.cat([self._stats[k], v], dim=0)
            elif isinstance(v, np.ndarray):
                self._stats[k] = np.concatenate([self._stats[k], v], axis=0)
            elif isinstance(v, list):
                self._stats[k] = self._stats[k] + deepcopy(v)
            else:
                raise TypeError(f'MaskData key {k} has an unsupported type {type(v)}.')

    def to_numpy(self) -> None:
        for k, v in self._stats.items():
            if isinstance(v, torch.Tensor):
                self._stats[k] = v.detach().cpu().numpy()


def is_box_near_crop_edge(boxes, crop_box, orig_box, atol: float = 20.0):
    crop_box_torch = torch.as_tensor(crop_box, dtype=torch.float, device=boxes.device)
    orig_box_torch = torch.as_tensor(orig_box, dtype=torch.float, device=boxes.device)
    boxes = uncrop_boxes_xyxy(boxes, crop_box).float()
    near_crop_edge = torch.isclose(boxes, crop_box_torch[None, :], atol=atol, rtol=0)
    near_image_edge = torch.isclose(boxes, orig_box_torch[None, :], atol=atol, rtol=0)
    near_crop_edge = torch.logical_and(near_crop_edge, ~near_image_edge)
    return torch.any(near_crop_edge, dim=1)


def box_xyxy_to_xywh(box_xyxy):
    box_xywh = deepcopy(box_xyxy)
    box_xywh[2] = box_xywh[2] - box_xywh[0]
    box_xywh[3] = box_xywh[3] - box_xywh[1]
    return box_xywh


def batch_iterator(batch_size: int, *args) -> Generator[List[Any], None, None]:
    assert len(args) > 0 and all(len(a) == len(args[0]) for a in args), 'Batched iteration must have inputs of all the same size.'
    n_batches = len(args[0]) // batch_size + int(len(args[0]) % batch_size != 0)
    for b in range(n_batches):
        yield [arg[b * batch_size:(b + 1) * batch_size] for arg in args]


def calculate_stability_score(masks, mask_threshold: float, threshold_offset: float):
    intersections = (masks > (mask_threshold + threshold_offset)).sum(-1, dtype=torch.int16).sum(-1, dtype=torch.int32)
    unions = (masks > (mask_threshold - threshold_offset)).sum(-1, dtype=torch.int16).sum(-1, dtype=torch.int32)
    return intersections / unions


def build_point_grid(n_per_side: int) -> np.ndarray:
    offset = 1 / (2 * n_per_side)
    points_one_side = np.linspace(offset, 1 - offset, n_per_side)
    points_x = np.tile(points_one_side[None, :], (n_per_side, 1))
    points_y = np.tile(points_one_side[:, None], (1, n_per_side))
    return np.stack([points_x, points_y], axis=-1).reshape(-1, 2)


def build_all_layer_point_grids(n_per_side: int, n_layers: int, scale_per_layer: int) -> List[np.ndarray]:
    return [build_point_grid(int(n_per_side / (scale_per_layer ** i))) for i in range(n_layers + 1)]


def generate_crop_boxes(im_size: Tuple[int, ...], n_layers: int, overlap_ratio: float):
    crop_boxes, layer_idxs = [], []
    im_h, im_w = im_size
    short_side = min(im_h, im_w)
    crop_boxes.append([0, 0, im_w, im_h])
    layer_idxs.append(0)

    def crop_len(orig_len, n_crops, overlap):
        return int(math.ceil((overlap * (n_crops - 1) + orig_len) / n_crops))

    for i_layer in range(n_layers):
        n_crops_per_side = 2 ** (i_layer + 1)
        overlap = int(overlap_ratio * short_side * (2 / n_crops_per_side))
        crop_w = crop_len(im_w, n_crops_per_side, overlap)
        crop_h = crop_len(im_h, n_crops_per_side, overlap)
        crop_box_x0 = [int((crop_w - overlap) * i) for i in range(n_crops_per_side)]
        crop_box_y0 = [int((crop_h - overlap) * i) for i in range(n_crops_per_side)]
        for x0 in crop_box_x0:
            for y0 in crop_box_y0:
                crop_boxes.append([x0, y0, min(x0 + crop_w, im_w), min(y0 + crop_h, im_h)])
                layer_idxs.append(i_layer + 1)
    return crop_boxes, layer_idxs


def uncrop_boxes_xyxy(boxes, crop_box: List[int]):
    x0, y0, _, _ = crop_box
    offset = torch.tensor([[x0, y0, x0, y0]], device=boxes.device)
    if len(boxes.shape) == 3:
        offset = offset.unsqueeze(1)
    return boxes + offset


def uncrop_points(points, crop_box: List[int]):
    x0, y0, _, _ = crop_box
    offset = torch.tensor([[x0, y0]], device=points.device)
    if len(points.shape) == 3:
        offset = offset.unsqueeze(1)
    return points + offset


def uncrop_masks(masks, crop_box: List[int], orig_h: int, orig_w: int):
    x0, y0, x1, y1 = crop_box
    if x0 == 0 and y0 == 0 and x1 == orig_w and y1 == orig_h:
        return masks
    pad_x, pad_y = orig_w - (x1 - x0), orig_h - (y1 - y0)
    pad = (x0, pad_x - x0, y0, pad_y - y0)
    return torch.nn.functional.pad(masks, pad, value=0)


def batched_mask_to_box(masks):
    if torch.numel(masks) == 0:
        return torch.zeros(*masks.shape[:-2], 4, device=masks.device)
    shape = masks.shape
    h, w = shape[-2:]
    if len(shape) > 2:
        masks = masks.flatten(0, -3)
    else:
        masks = masks.unsqueeze(0)
    in_height, _ = torch.max(masks, dim=-1)
    in_height_coords = in_height * torch.arange(h, device=in_height.device)[None, :]
    bottom_edges, _ = torch.max(in_height_coords, dim=-1)
    in_height_coords = in_height_coords + h * (~in_height)
    top_edges, _ = torch.min(in_height_coords, dim=-1)
    in_width, _ = torch.max(masks, dim=-2)
    in_width_coords = in_width * torch.arange(w, device=in_width.device)[None, :]
    right_edges, _ = torch.max(in_width_coords, dim=-1)
    in_width_coords = in_width_coords + w * (~in_width)
    left_edges, _ = torch.min(in_width_coords, dim=-1)
    empty_filter = (right_edges < left_edges) | (bottom_edges < top_edges)
    out = torch.stack([left_edges, top_edges, right_edges, bottom_edges], dim=-1)
    out = out * (~empty_filter).unsqueeze(-1)
    if len(shape) > 2:
        out = out.reshape(*shape[:-2], 4)
    else:
        out = out[0]
    return out


def _unsupported(*args, **kwargs):
    raise NotImplementedError('RLE output and small-region removal are not part of the stand-in segment_anything')


mask_to_rle_pytorch = rle_to_mask = area_from_rle = coco_encode_rle = remove_small_regions = _unsupported

# ------------------------------------------------------------------------------------- utils/transforms.py


class ResizeLongestSide:
    def __init__(self, target_length: int) -> None:
        self.target_length = target_length

    def apply_image(self, image: np.ndarray) -> np.ndarray:
        from PIL import Image
        target_size = self.get_preprocess_shape(image.shape[0], image.shape[1], self.target_length)
        return np.array(Image.fromarray(image).resize(target_size[::-1], Image.BILINEAR))

    def apply_coords(self, coords: np.ndarray, original_size: Tuple[int, ...]) -> np.ndarray:
        old_h, old_w = original_size
        new_h, new_w = self.get_preprocess_shape(original_size[0], original_size[1], self.target_length)
        coords = deepcopy(coords).astype(float)
        coords[..., 0] = coords[..., 0] * (new_w / old_w)
        coords[..., 1] = coords[..., 1] * (new_h / old_h)
        return coords

    @staticmethod
    def get_preprocess_shape(oldh: int, oldw: int, long_side_length: int) -> Tuple[int, int]:
        scale = long_side_length * 1.0 / max(oldh, oldw)
        newh, neww = oldh * scale, oldw * scale
        return (int(newh + 0.5), int(neww + 0.5))

# --------------------------------------------------------------------------------------- modeling/sam.py


class Sam(torch.nn.Module):
    mask_threshold: float = 0.0
    image_format: str = 'RGB'

    def __init__(self, image_encoder, prompt_encoder, mask_decoder) -> None:
        super().__init__()
        self.image_encoder = image_encoder
        self.prompt_encoder = prompt_encoder
        self.mask_decoder = mask_decoder
        self.register_buffer('pixel_mean', torch.Tensor([123.675, 116.28, 103.53]).view(-1, 1, 1), False)
        self.register_buffer('pixel_std', torch.Tensor([58.395, 57.12, 57.375]).view(-1, 1, 1), False)

    @property
    def device(self) -> Any:
        return self.pixel_mean.device

    def postprocess_masks(self, masks, input_size: Tuple[int, ...], original_size: Tuple[int, ...]):
        masks = F.interpolate(masks, (self.image_encoder.img_size, self.image_encoder.img_size), mode='bilinear',
                              align_corners=False)
        masks = masks[..., :input_size[0], :input_size[1]]
        return F.interpolate(masks, original_size, mode='bilinear', align_corners=False)

    def preprocess(self, x):
        x = (x - self.pixel_mean) / self.pixel_std
        h, w = x.shape[-2:]
        padh = self.image_encoder.img_size - h
        padw = self.image_encoder.img_size - w
        return F.pad(x, (0, padw, 0, padh))

# ----------------------------------------------------------------------------------------------- predictor.py


class SamPredictor:
    def __init__(self, sam_model: Sam) -> None:
        super().__init__()
        self.model = sam_model
        self.transform = ResizeLongestSide(sam_model.image_encoder.img_size)
        self.reset_image()

    def set_image(self, image: np.ndarray, image_format: str = 'RGB') -> None:
        assert image_format in ['RGB', 'BGR'], f"image_format must be in ['RGB', 'BGR'], is {image_format}."
        if image_format != self.model.image_format:
            image = image[..., ::-1]
        input_image = self.transform.apply_image(image)
        input_image_torch = torch.as_tensor(input_image, device=self.device)
        input_image_torch = input_image_torch.permute(2, 0, 1).contiguous()[None, :, :, :]
        self.set_torch_image(input_image_torch, image.shape[:2])

    @torch.no_grad()
    def set_torch_image(self, transformed_image, original_image_size: Tuple[int, ...]) -> None:
        assert (len(transformed_image.shape) == 4 and transformed_image.shape[1] == 3
                and max(*transformed_image.shape[2:]) == self.model.image_encoder.img_size)
        self.reset_image()
        self.original_size = original_image_size
        self.input_size = tuple(transformed_image.shape[-2:])
        input_image = self.model.preprocess(transformed_image)
        self.features = self.model.image_encoder(input_image)
        self.is_image_set = True

    @torch.no_grad()
    def predict_torch(self, point_coords, point_labels, boxes=None, mask_input=None, multimask_output: bool = True,
                      return_logits: bool = False):
        if not self.is_image_set:
            raise RuntimeError('An image must be set with .set_image(...) before mask prediction.')
        points = (point_coords, point_labels) if point_coords is not None else None
        sparse_embeddings, dense_embeddings = self.model.prompt_encoder(points=points, boxes=boxes, masks=mask_input)
        low_res_masks, iou_predictions = self.model.mask_decoder(
            image_embeddings=self.features,
            image_pe=self.model.prompt_encoder.get_dense_pe(),
            sparse_prompt_embeddings=sparse_embeddings,
            dense_prompt_embeddings=dense_embeddings,
            multimask_output=multimask_output,
        )
        masks = self.model.postprocess_masks(low_res_masks, self.input_size, self.original_size)
        if not return_logits:
            masks = masks > self.model.mask_threshold
        return masks, iou_predictions, low_res_masks

    @property
    def device(self):
        return self.model.device

    def reset_image(self) -> None:
        self.is_image_set = False
        self.features = None
        self.orig_h = self.orig_w = self.input_h = self.input_w = None

# ------------------------------------------------------------------------------------------- the fake model


class _Encoder(torch.nn.Module):
    img_size = 1024

    def forward(self, x):
        return x.mean(dim=(2, 3), keepdim=True)


class _PromptEncoder(torch.nn.Module):
    """Passes the prompts through: sparse = [B, P, 3] float32 (x, y, label) in input coordinates."""

    def forward(self, points, boxes, masks):
        coords, labels = points
        sparse = torch.cat([coords.float(), labels[..., None].float()], dim=-1)
        return sparse, torch.zeros(1, device=sparse.device)

    def get_dense_pe(self):
        return torch.zeros(1)


def _hash(key, salt):
    return torch.frac(torch.sin(key * 12.9898 + salt * 78.233) * 43758.5453).abs()


class _MaskDecoder(torch.nn.Module):
    def __init__(self, seed: int, low_iou_top: float, dead: float) -> None:
        super().__init__()
        self.seed, self.low_iou_top, self.dead = seed, low_iou_top, dead

    def forward(self, image_embeddings, image_pe, sparse_prompt_embeddings, dense_prompt_embeddings,
                multimask_output):
        pts = sparse_prompt_embeddings.double()
        dev = pts.device
        b = pts.shape[0]
        x, y = pts[:, 0, 0], pts[:, 0, 1]  # the positive prompt, input coordinates
        k = torch.arange(3, device=dev, dtype=torch.float64)
        key = (torch.floor(x * 8) * 0.0131 + torch.floor(y * 8) * 0.0371 + self.seed * 1.618)[:, None] + k * 0.7071
        radius = 3 + 45 * _hash(key, 1)                    # low-res pixels
        slope = 0.35 + 5 * _hash(key, 2) ** 2
        iou = torch.round((0.80 + 0.2 * _hash(key, 3)) * 32) / 32
        aspect = 0.7 + 0.6 * _hash(key, 4)
        phase = 6.283 * _hash(key, 5)
        dead = _hash(key, 6) < self.dead
        iou = torch.where(dead, torch.full_like(iou, 0.96875), iou)
        iou = torch.where((y < self.low_iou_top * 1024)[:, None], torch.full_like(iou, 0.5), iou)
        g = torch.arange(256, device=dev, dtype=torch.float64)
        gy, gx = g.view(1, 1, 256, 1), g.view(1, 1, 1, 256)
        cy, cx = (y / 4 - 0.5).view(b, 1, 1, 1), (x / 4 - 0.5).view(b, 1, 1, 1)
        d = torch.sqrt(((gx - cx) * aspect.view(b, 3, 1, 1)) ** 2 + (gy - cy) ** 2)
        logits = slope.view(b, 3, 1, 1) * (radius.view(b, 3, 1, 1) - d)
        logits = logits + 0.3 * torch.sin(gx / 9 + phase.view(b, 3, 1, 1)) * torch.cos(gy / 11)
        for p in range(1, pts.shape[1]):  # negative prompts carve a hole
            ny, nx = (pts[:, p, 1] / 4 - 0.5).view(b, 1, 1, 1), (pts[:, p, 0] / 4 - 0.5).view(b, 1, 1, 1)
            hole = torch.clamp(8 - torch.sqrt((gx - nx) ** 2 + (gy - ny) ** 2), min=0)
            logits = logits - 3 * hole * (pts[:, p, 2] == 0).view(b, 1, 1, 1)
        logits = torch.where(dead.view(b, 3, 1, 1), -1.5 - 0.4 * torch.sigmoid(logits), logits)
        return logits.float(), iou.float()


class FakeSam(Sam):
    """seed: varies the masks; low_iou_top: prompts in the top fraction of the input get predicted IoU 0.5 (whole
    batches filtered); dead: fraction of masks entirely below -1 with a high predicted IoU."""

    def __init__(self, seed: int = 0, low_iou_top: float = 0.0, dead: float = 0.04) -> None:
        super().__init__(_Encoder(), _PromptEncoder(), _MaskDecoder(seed, low_iou_top, dead))


# a build_sam-style registry for deva.ext.automatic_sam.get_sam_model: config SAM_ENCODER_VERSION 'fake' builds FakeSam()
sam_model_registry = {'fake': lambda checkpoint=None: FakeSam()}

# ----------------------------------------------------------------------------------------------- installing
_MODULES = ('segment_anything', 'segment_anything.modeling', 'segment_anything.predictor', 'segment_anything.utils',
            'segment_anything.utils.amg', 'segment_anything.utils.transforms')


def install() -> dict:
    """Make ``import segment_anything...`` resolve to this stand-in; returns the modules it replaced."""
    me = sys.modules[__name__]
    saved = {name: sys.modules.get(name) for name in _MODULES}
    mods = {name: types.ModuleType(name) for name in _MODULES}
    mods['segment_anything'].__path__ = []
    mods['segment_anything.utils'].__path__ = []
    mods['segment_anything.modeling'].Sam = Sam
    mods['segment_anything.predictor'].SamPredictor = SamPredictor
    mods['segment_anything'].SamPredictor = SamPredictor
    mods['segment_anything'].sam_model_registry = sam_model_registry
    mods['segment_anything.utils.transforms'].ResizeLongestSide = ResizeLongestSide
    amg = mods['segment_anything.utils.amg']
    for name in ('MaskData', 'area_from_rle', 'batch_iterator', 'batched_mask_to_box', 'box_xyxy_to_xywh',
                 'build_all_layer_point_grids', 'build_point_grid', 'calculate_stability_score', 'coco_encode_rle',
                 'generate_crop_boxes', 'is_box_near_crop_edge', 'mask_to_rle_pytorch', 'remove_small_regions',
                 'rle_to_mask', 'uncrop_boxes_xyxy', 'uncrop_masks', 'uncrop_points'):
        setattr(amg, name, getattr(me, name))
    for name in ('modeling', 'predictor', 'utils'):
        setattr(mods['segment_anything'], name, mods[f'segment_anything.{name}'])
    mods['segment_anything.utils'].amg = amg
    mods['segment_anything.utils'].transforms = mods['segment_anything.utils.transforms']
    sys.modules.update(mods)
    return saved


def uninstall(saved: dict) -> None:
    for name, mod in saved.items():
        if mod is None:
            sys.modules.pop(name, None)
        else:
            sys.modules[name] = mod
