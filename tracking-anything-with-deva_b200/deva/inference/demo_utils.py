"""Drop-in for the reference's deva/inference/demo_utils.py: the demos' per-frame ingest on the device.

``get_input_frame_for_deva`` uploads the uint8 frame as is (3 bytes per pixel, through pinned memory, without a host
synchronisation) or takes a frame already on the device (``DeviceLoader`` over a ``SimpleVideoReader``), and normalises
and resizes it there with ``frame_io.frame_from_rgb8(..., resize='demo')``: the reference's float32 conversion,
``im_normalization`` and plain bilinear ``F.interpolate``, run on the host before ``.cuda()``.  Importing this module
does not initialise CUDA and needs no ``deva.dataset``.
"""
import numpy as np
import torch

from deva.inference.frame_io import frame_from_rgb8


def get_input_frame_for_deva(image_np, min_side: int) -> torch.Tensor:
    """image_np: uint8 [H, W, 3] RGB, a numpy array or a CUDA tensor.  -> normalised float32 [3, H', W'] on the current
    CUDA device, the short side resized to ``min_side`` (the demo's int(h * scale), int(w * scale); min_side <= 0:
    H, W): the reference's frame within 1e-6, and bit for bit without a resize."""
    if isinstance(image_np, np.ndarray):
        if image_np.dtype != np.uint8 or image_np.ndim != 3 or image_np.shape[2] != 3:
            raise TypeError(f'get_input_frame_for_deva takes a uint8 [H, W, 3] frame, got a {image_np.dtype} array '
                            f'of shape {image_np.shape}')
        frame = torch.from_numpy(np.ascontiguousarray(image_np)).pin_memory()
    elif isinstance(image_np, torch.Tensor) and image_np.is_cuda:
        if image_np.dtype != torch.uint8 or image_np.dim() != 3 or image_np.shape[2] != 3:
            raise TypeError(f'get_input_frame_for_deva takes a uint8 [H, W, 3] frame, got a {image_np.dtype} CUDA '
                            f'tensor of shape {tuple(image_np.shape)}')
        frame = image_np
    else:
        kind = f'a {image_np.device} tensor' if isinstance(image_np, torch.Tensor) else type(image_np).__name__
        raise TypeError(f'get_input_frame_for_deva takes a numpy array or a CUDA tensor, got {kind}')
    return frame_from_rgb8(frame, size=min_side if min_side > 0 else None, resize='demo',
                           device=torch.device('cuda', torch.cuda.current_device()))


@torch.inference_mode()
def flush_buffer(deva, result_saver) -> None:
    """Steps and saves the frames left in ``deva``'s semi-online buffer (the reference's, for numpy or CUDA frames)."""
    cfg = deva.config
    new_min_side = cfg['size']
    need_resize = new_min_side > 0

    if 'prompt' in cfg:
        prompts = cfg['prompt'].split('.')
    else:
        prompts = None

    for frame_info in deva.frame_buffer:
        this_image = frame_info.image
        this_frame_name = frame_info.name
        this_image_np = frame_info.image_np
        h, w = (int(v) for v in this_image_np.shape[:2])
        prob = deva.step(this_image, None, None)
        result_saver.save_mask(prob,
                               this_frame_name,
                               need_resize=need_resize,
                               shape=(h, w),
                               image_np=this_image_np,
                               prompts=prompts)
