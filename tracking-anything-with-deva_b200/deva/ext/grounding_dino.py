"""Drop-in for the reference's deva/ext/grounding_dino.py: Grounding-DINO boxes prompted into SAM -> detection id map on
the device.

The detector packages (``groundingdino``, ``segment_anything``, ``deva.ext.MobileSAM`` / ``LightHQSAM``) are imported by
``get_grounding_dino_model`` only, so importing this module needs none of them and does not initialise CUDA.
"""
from typing import Dict, List

import numpy as np
import torch

from deva.ext.detector_masks import cover_id_map, host_image, output_size, stack_masks
from deva.inference.object_info import ObjectInfo


def _grounding_dino_class():
    try:
        from groundingdino.util.inference import Model
    except ImportError:  # a source checkout of GroundingDINO next to the demo
        from GroundingDINO.groundingdino.util.inference import Model
    return Model


def get_grounding_dino_model(config: Dict, device: str):
    """-> (Grounding-DINO model, SamPredictor) for config['sam_variant'] in 'mobile', 'original', 'sam_hq' and
    'sam_hq_light'."""
    gd_model = _grounding_dino_class()(model_config_path=config['GROUNDING_DINO_CONFIG_PATH'],
                                       model_checkpoint_path=config['GROUNDING_DINO_CHECKPOINT_PATH'],
                                       device=device)
    from segment_anything import SamPredictor
    variant = config['sam_variant'].lower()
    if variant in ('mobile', 'sam_hq_light'):
        if variant == 'mobile':
            from deva.ext.MobileSAM.setup_mobile_sam import setup_model
            weights = torch.load(config['MOBILE_SAM_CHECKPOINT_PATH'])
        else:
            from deva.ext.LightHQSAM.setup_light_hqsam import setup_model
            weights = torch.load(config['LIGHT_HQ_SAM_CHECKPOINT_PATH'])
        model = setup_model()
        model.load_state_dict(weights, strict=True)
        model.to(device=device)
    elif variant == 'original':
        from segment_anything import sam_model_registry
        model = sam_model_registry[config['SAM_ENCODER_VERSION']](checkpoint=config['SAM_CHECKPOINT_PATH']).to(
            device=device)
    elif variant == 'sam_hq':
        from segment_anything import sam_hq_model_registry
        model = sam_hq_model_registry[config['SAM_ENCODER_VERSION']](checkpoint=config['HQ_SAM_CHECKPOINT_PATH']).to(
            device=device)
    else:
        raise ValueError(f'Unknown SAM variant: {config["sam_variant"]}')
    return gd_model, SamPredictor(model)


def segment_with_text(config: Dict, gd_model, sam, image: np.ndarray, prompts: List[str],
                      min_side: int) -> (torch.Tensor, List[ObjectInfo]):
    """image: H*W*3 uint8 RGB (0~255), a numpy array or a CUDA tensor; prompts: class names.

    Returns the int64 id map at the working resolution (shorter side ``min_side``; the image size when min_side <= 0)
    on the detector's device, and one ObjectInfo(id, category_id=class id, score=confidence) per painted mask.  SAM and
    Grounding-DINO are given the host array: a CUDA image is downloaded once into pinned memory, a host
    synchronisation on top of the one the id map needs."""
    import cv2
    import torchvision

    image = host_image(image)
    threshold = config['DINO_THRESHOLD']
    sam.set_image(image, image_format='RGB')
    detections = gd_model.predict_with_classes(image=cv2.cvtColor(image, cv2.COLOR_RGB2BGR), classes=prompts,
                                               box_threshold=threshold, text_threshold=threshold)
    keep = torchvision.ops.nms(torch.from_numpy(detections.xyxy), torch.from_numpy(detections.confidence),
                               config['DINO_NMS_THRESHOLD']).numpy().tolist()
    detections.xyxy = detections.xyxy[keep]
    detections.confidence = detections.confidence[keep]
    detections.class_id = detections.class_id[keep]

    result_masks = []
    for box in detections.xyxy:
        masks, scores, _ = sam.predict(box=box, multimask_output=True)
        result_masks.append(masks[np.argmax(scores)])
    detections.mask = stack_masks(result_masks)

    new_h, new_w = output_size(*image.shape[:2], min_side)
    id_map, segments = cover_id_map(detections.mask, new_h, new_w, gd_model.device)
    return id_map, [ObjectInfo(id=i, category_id=detections.class_id[k], score=detections.confidence[k])
                    for i, k in segments]
