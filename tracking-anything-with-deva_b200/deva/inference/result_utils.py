"""Drop-in ``ResultSaver`` (surface and outputs of the reference's deva/inference/result_utils.py) whose per-frame pixel
work runs on the device.

``save_mask`` runs ``frame_io.prob_to_segments`` on the current stream - resize, argmax, id remap, uint8 / RGB id image,
overlay, per-channel areas and boxes in one kernel - starts the device-to-host copies into a ring of pinned buffers,
records an event and queues the frame; it never synchronises the host.  The writer thread waits on the event and does
only what has to stay on the host: PIL images and PNG / JPEG encoding, the JSON entries, the gradio writer, and the two
paths that need third-party code - ``supervision`` boxes and labels for prompts, and ``pycocotools`` RLE for burst (a
full-frame compare and encode per segment, from the downloaded id map).  Both libraries are imported only when those
paths run.

With ``png_encoder='device'`` (or ``DEVA_B200_PNG_ENCODER=device``) the id image is encoded as a PNG on the device too
(deva/utils/png_encode.py), right after ``prob_to_segments`` on the same stream: only the compressed stream comes to the
host, and the writer thread writes its bytes.  The files decode to the pixels, mode and palette Pillow's files decode to.

With ``jpeg_encoder='device'`` (or ``DEVA_B200_JPEG_ENCODER=device``) the demo overlay JPEG is encoded on the device
(deva/utils/jpeg_encode.py), byte for byte Pillow's file.  An overlay blended on the device is encoded right after
``prob_to_segments`` and only its scan comes to the host; an image finished on the host (prompt boxes and labels, or
the host blend) is encoded by the writer thread.  The gradio writer is unchanged.

With ``rle_encoder='device'`` (or ``DEVA_B200_RLE_ENCODER=device``) burst's per-segment COCO RLE is encoded on the
device (deva/utils/rle_encode.py), string for string pycocotools': every segment's string comes from one pass over the
id map right after ``prob_to_segments``, and only the strings come to the host, not the id map.  The writer builds the
same JSON entries from them, with no per-segment pixel work and no pycocotools.

With ``jpeg_decoder='device'`` (or ``DEVA_B200_JPEG_DECODER=device``) an overlay given as ``path_to_image`` (no
``image_np``) is blended on the device too: ``save_mask`` reads the file, and when it is a device-eligible JPEG
(deva/utils/jpeg_decode.py) of the output size it decodes it on the current stream and feeds it to
``prob_to_segments(frame=...)``, as it does with ``image_np``.  Whether the device accepted the file is known only to the
writer, through a status downloaded with the frame's other copies; on a nonzero status the writer makes exactly what
the Pillow path makes - Pillow's decode and the host blend - from the frame's device id map and RGB id image, which the
queued frame keeps referenced and downloads only then.  A file that cannot be read, does not parse or has another size
takes the Pillow path as before.

``image_np`` may also be a CUDA uint8 [h, w, 3] tensor of the output size (a frame the demos read on the device): it is
blended as it is, with no staging copy, and the queued frame keeps it referenced until its copies are done; everything
after the blend is the numpy ``image_np`` path.  A CUDA ``image_np`` of another shape or dtype is copied to pinned memory
with the frame's other downloads and the writer treats it as that numpy array.
"""
import copy
import os
from dataclasses import dataclass
from os import path
from queue import Queue
from threading import Thread
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
from PIL import Image

from deva.inference.frame_io import prob_to_ids, prob_to_segments
from deva.utils import jpeg_decode
from deva.utils.device_decode import read_bytes
from deva.utils.device_download import Pending, write
from deva.utils.jpeg_encode import encode_jpeg_async, host_bytes as jpeg_host_bytes
from deva.utils.jpeg_encode import resolve_encoder as resolve_jpeg_encoder
from deva.utils.png_encode import encode_png_async, host_bytes as png_host_bytes, resolve_encoder
from deva.utils.rle_encode import MAX_SEGMENT_CHANNELS, encode_rle_async, host_bytes as rle_host_bytes
from deva.utils.rle_encode import resolve_encoder as resolve_rle_encoder

QUEUE_SIZE = 10
RING_SIZE = QUEUE_SIZE + 2  # the queued frames, the one the writer holds and the one save_mask is filling


class ResultSaver:
    def __init__(self, output_root: str, video_name: str, *, dataset: str, object_manager, palette=None,
                 png_encoder: Optional[str] = None, jpeg_encoder: Optional[str] = None,
                 rle_encoder: Optional[str] = None, jpeg_decoder: Optional[str] = None):
        """png_encoder: 'pil' (Pillow on the writer thread) or 'device'; None reads DEVA_B200_PNG_ENCODER (default
        'pil').  jpeg_encoder: the same for the overlay JPEG; None reads DEVA_B200_JPEG_ENCODER (default 'pil').
        rle_encoder: 'pycocotools' (on the writer thread) or 'device' for burst's RLE; None reads DEVA_B200_RLE_ENCODER
        (default 'pycocotools').  jpeg_decoder: 'pil' (Pillow on the writer thread) or 'device' for an overlay's
        ``path_to_image``; None reads DEVA_B200_JPEG_DECODER (default 'pil')."""
        self.output_root = output_root
        self.png_encoder = resolve_encoder(png_encoder)
        self.jpeg_encoder = resolve_jpeg_encoder(jpeg_encoder)
        self.rle_encoder = resolve_rle_encoder(rle_encoder)
        self.jpeg_decoder = jpeg_decode.resolve_decoder(jpeg_decoder)
        self.video_name = video_name
        self.dataset = dataset.lower()
        self.palette = palette
        self.object_manager = object_manager

        self.need_remapping = False
        self.json_style = None
        self.output_postfix = None
        self.visualize = False

        if self.dataset == 'vipseg':
            self.all_annotations = []
            self.video_json = {'video_id': video_name, 'annotations': self.all_annotations}
            self.need_remapping = True
            self.json_style = 'vipseg'
            self.output_postfix = 'pan_pred'
        elif self.dataset == 'burst':
            self.need_remapping = True
            self.all_annotations = []
            self.video_json = {
                'dataset': path.dirname(video_name),
                'seq_name': path.basename(video_name),
                'segmentations': self.all_annotations
            }
            self.json_style = 'burst'
        elif self.dataset == 'unsup_davis17':
            self.need_remapping = True
        elif self.dataset == 'ref_davis':
            pass
        elif self.dataset == 'demo':
            self.need_remapping = True
            self.all_annotations = []
            self.video_json = {'annotations': self.all_annotations}
            self.json_style = 'vipseg'
            self.visualize = True
            self.visualize_postfix = 'Visualizations'
            self.output_postfix = 'Annotations'
        elif self.dataset == 'gradio':
            # minimal mode: a cv2.VideoWriter is expected to be assigned to self.writer
            self.writer = None
            self.need_remapping = True
            self.visualize = True
        else:
            raise NotImplementedError

        self.free_slots = Queue()
        for _ in range(RING_SIZE):
            self.free_slots.put({})
        self.queue = Queue(maxsize=QUEUE_SIZE)
        self.thread = Thread(target=save_result, args=(self.queue, ))
        self.thread.daemon = True
        self.thread.start()

    def save_mask(self,
                  prob: torch.Tensor,
                  frame_name: str,
                  need_resize: bool = False,
                  shape: Optional[Tuple[int, int]] = None,
                  save_the_mask: bool = True,
                  image_np: np.ndarray = None,
                  prompts: List[str] = None,
                  path_to_image: str = None):
        prob = prob.float()
        size = (int(shape[0]), int(shape[1])) if need_resize else tuple(prob.shape[-2:])
        long_id = self.object_manager.use_long_id
        overlay = save_the_mask and self.visualize and long_id
        on_device = (isinstance(image_np, np.ndarray) and image_np.dtype == np.uint8 and image_np.shape == (*size, 3))
        cuda_image = isinstance(image_np, torch.Tensor) and image_np.is_cuda
        if cuda_image:
            on_device = image_np.dtype == torch.uint8 and tuple(image_np.shape) == (*size, 3)
        if overlay and image_np is None and path_to_image is None:
            raise ValueError('Cannot visualize without image_np or path_to_image')

        header = None
        if overlay and image_np is None and path_to_image is not None and self.jpeg_decoder == 'device':
            data = read_bytes(path_to_image)
            header = None if data is None else jpeg_decode.parse(data)
            if header is not None and header.shape != (*size, 3):
                header = None

        slot = self.free_slots.get()  # blocks only while every slot is queued or being written
        frame = decoded = None
        if overlay and on_device and cuda_image:
            frame = image_np
        elif overlay and on_device:
            staged = _pinned(slot, 'image', image_np.shape, torch.uint8)
            staged.numpy()[...] = image_np
            frame = staged.to(prob.device, non_blocking=True)
        elif header is not None:
            frame, status, keep = jpeg_decode.decode_async(header)
            decoded = Decoded(status, keep)
            on_device = True  # the blend, its encoding and its downloads take the image_np path
        seg = prob_to_segments(prob, self.object_manager, size, index=save_the_mask and not long_id,
                               rgb=save_the_mask and long_id, frame=frame,
                               stats=self.json_style is not None or self.visualize, remap=self.need_remapping)
        png = None
        if save_the_mask and self.png_encoder == 'device' and self.dataset != 'gradio':
            png = encode_png_async(seg.rgb if long_id else seg.index,
                                   'RGB' if long_id else 'L' if self.palette is None else 'P', self.palette,
                                   host=_pinned(slot, 'png', (png_host_bytes(), ), torch.uint8))
        jpeg = None
        if overlay and on_device and prompts is None and self.jpeg_encoder == 'device' and self.dataset != 'gradio':
            jpeg = encode_jpeg_async(seg.overlay, host=_pinned(slot, 'jpeg', (jpeg_host_bytes(), ), torch.uint8))
        host = {}
        for name in ('index', 'rgb', 'overlay', 'counts', 'boxes'):
            t = getattr(seg, name)
            # an encoded id image stays on the device; the host blend still needs the RGB ids
            if png is not None and (name == 'index' or (name == 'rgb' and not (overlay and not on_device))):
                continue
            if jpeg is not None and name == 'overlay':  # an encoded overlay stays on the device
                continue
            if t is not None:
                host[name] = _pinned(slot, name, t.shape, t.dtype)
                host[name].copy_(t, non_blocking=True)
        if overlay and cuda_image and not on_device:  # the writer blends it as the numpy array the reference got
            host['image_np'] = _pinned(slot, 'image_np', image_np.shape, image_np.dtype)
            host['image_np'].copy_(image_np, non_blocking=True)
        segments_info = copy.deepcopy(self.object_manager.get_current_segments_info())
        rle = None
        if self.json_style == 'burst' or (overlay and not on_device):
            # the full id map: burst's per-segment RLE and the host blend need ids, not colours
            lut = torch.tensor(seg.lut, dtype=torch.int32).pin_memory().to(prob.device, non_blocking=True)
            ids = prob_to_ids(prob, size=size, lut=lut)
            if self.json_style == 'burst' and self.rle_encoder == 'device':
                rle = encode_rle_async(ids, [s['id'] for s in segments_info],
                                       host=_pinned(slot, 'rle', (rle_host_bytes(MAX_SEGMENT_CHANNELS), ), torch.uint8))
            if rle is None or (overlay and not on_device):  # encoded RLE strings replace the id map's download
                host['ids'] = _pinned(slot, 'ids', ids.shape, ids.dtype)
                host['ids'].copy_(ids, non_blocking=True)
        if decoded is not None:
            # what a declined file's host blend needs, kept on the device and downloaded only then
            lut = torch.tensor(seg.lut, dtype=torch.int32).pin_memory().to(prob.device, non_blocking=True)
            decoded.ids, decoded.rgb, decoded.frame = prob_to_ids(prob, size=size, lut=lut), seg.rgb, frame
            host['jpeg_status'] = _pinned(slot, 'jpeg_status', (1, ), torch.int32)
            host['jpeg_status'].copy_(decoded.status, non_blocking=True)
        done = torch.cuda.Event()
        done.record()

        self.queue.put(ResultArgs(
            saver=self,
            slot=slot,
            host=host,
            done=done,
            lut=seg.lut,
            long_id=long_id,
            frame_name=frame_name,
            save_the_mask=save_the_mask,
            image_np=None if on_device or cuda_image else image_np,
            frame=frame if cuda_image else None,
            decoded=decoded,
            prompts=prompts,
            path_to_image=path_to_image,
            all_obj_ids=[int(o.id) for o in self.object_manager.obj_to_tmp_id],
            segments_info=segments_info,
            png=png,
            jpeg=jpeg,
            rle=rle,
        ))

    def end(self):
        self.queue.put(None)
        self.queue.join()
        self.thread.join()


def _pinned(slot: Dict[str, torch.Tensor], name: str, shape, dtype) -> torch.Tensor:
    """The slot's pinned buffer ``name``, reallocated when the shape or dtype changes."""
    t = slot.get(name)
    if t is None or t.shape != shape or t.dtype != dtype:
        t = slot[name] = torch.empty(shape, dtype=dtype, pin_memory=True)
    return t


@dataclass
class Decoded:
    """A ``path_to_image`` JPEG decoded on the device: its status, and what stays referenced until the writer is done -
    the decode's buffers, the frame, and the id map and RGB id image a declined file's host blend downloads."""
    status: torch.Tensor
    keep: object
    ids: Optional[torch.Tensor] = None
    rgb: Optional[torch.Tensor] = None
    frame: Optional[torch.Tensor] = None


@dataclass
class ResultArgs:
    saver: ResultSaver
    slot: Dict[str, torch.Tensor]  # pinned ring slot, returned to saver.free_slots when written
    host: Dict[str, torch.Tensor]  # views of the slot's buffers that this frame's copies fill
    done: torch.cuda.Event  # recorded after the copies
    lut: List[int]  # prob channel -> id written for it
    long_id: bool
    frame_name: str
    save_the_mask: bool
    image_np: np.ndarray  # only when the overlay is blended on the host
    prompts: List[str]
    path_to_image: str
    all_obj_ids: List[int]
    segments_info: List[Dict]
    png: Optional[Pending] = None  # the id image's PNG, encoded on the device
    jpeg: Optional[Pending] = None  # the overlay's JPEG, encoded on the device
    rle: Optional[Pending] = None  # burst's RLE of every entry of segments_info, encoded on the device
    decoded: Optional[Decoded] = None  # path_to_image decoded on the device
    frame: Optional[torch.Tensor] = None  # a CUDA image_np blended as it is, referenced until the copies are done


def save_result(queue: Queue):
    while True:
        args: ResultArgs = queue.get()
        if args is None:
            queue.task_done()
            break
        args.done.synchronize()
        _write(args)
        args.saver.free_slots.put(args.slot)
        queue.task_done()


def _write(args: ResultArgs):
    saver, host, frame_name, segments_info = args.saver, args.host, args.frame_name, args.segments_info
    area, box = {}, {}
    if 'counts' in host:
        counts, boxes = host['counts'].tolist(), host['boxes'].tolist()
        for k, v in enumerate(args.lut):
            if counts[k] == 0:
                continue
            area[v] = area.get(v, 0) + counts[k]
            b = box.get(v, boxes[k])
            box[v] = [min(b[0], boxes[k][0]), min(b[1], boxes[k][1]), max(b[2], boxes[k][2]), max(b[3], boxes[k][3])]

    # record output in the json file
    if saver.json_style == 'vipseg':
        for seg in segments_info:
            seg['area'] = area.get(seg['id'], 0)
        segments_info = [s for s in segments_info if s['area'] > 0]
        saver.all_annotations.append({'file_name': frame_name[:-4] + '.jpg', 'segments_info': segments_info})
    elif saver.json_style == 'burst':
        if args.rle is not None:
            for seg, rle in zip(segments_info, args.rle.result()):
                seg['area'] = area.get(seg['id'], 0)
                seg['rle_mask'] = rle
        else:
            import pycocotools.mask as mask_util
            ids = host['ids'].numpy()
            for seg in segments_info:
                m = ids == seg['id']
                seg['area'] = area.get(seg['id'], 0)
                coco_mask = mask_util.encode(np.asfortranarray(m))
                coco_mask['counts'] = coco_mask['counts'].decode('utf-8')
                seg['rle_mask'] = coco_mask
        segments_info = [s for s in segments_info if s['area'] > 0]
        saver.all_annotations.append({
            'file_name': frame_name[:-4] + '.jpg',
            'segmentations': [{'id': s['id'], 'score': s['score'], 'rle': s['rle_mask']} for s in segments_info],
        })
    elif saver.visualize:
        for seg in segments_info:
            seg['area'] = area.get(seg['id'], 0)
        segments_info = [s for s in segments_info if s['area'] > 0]

    if not args.save_the_mask:
        return
    if args.png is not None:
        write(args.png, _path(saver, saver.output_postfix, frame_name[:-4] + '.png'))
    else:
        if args.long_id:
            out_img = Image.fromarray(host['rgb'].numpy())
        else:
            out_img = Image.fromarray(host['index'].numpy())
            if saver.palette is not None:
                out_img.putpalette(saver.palette)
        if saver.dataset != 'gradio':
            _save(out_img, saver, saver.output_postfix, frame_name[:-4] + '.png')

    if not (saver.visualize and args.long_id):
        return
    # a path_to_image the device declined: the device's overlay (and its JPEG) are discarded for Pillow's path
    declined = args.decoded is not None and int(host['jpeg_status'][0]) != 0
    if args.jpeg is not None and not declined:
        write(args.jpeg, _path(saver, saver.visualize_postfix, frame_name[:-4] + '.jpg'))
        return
    if 'overlay' in host and not declined:
        blend = host['overlay'].numpy()
    else:
        image_np = args.image_np
        if image_np is None and 'image_np' in host:
            image_np = host['image_np'].numpy()
        if image_np is None:
            image_np = np.array(Image.open(args.path_to_image))
        ids = args.decoded.ids.cpu().numpy() if declined else host['ids'].numpy()
        rgb = host['rgb'].numpy() if 'rgb' in host else args.decoded.rgb.cpu().numpy()
        # the reference's blend: alpha = 1 where the id is 0, else 0.5
        alpha = (ids == 0).astype(np.float32)[:, :, None] * 0.5 + 0.5
        blend = (image_np * alpha + rgb * (1 - alpha)).astype(np.uint8)

    if args.prompts is not None and len(segments_info) > 0:
        import supervision as sv
        labels = [f'{args.prompts[s["category_id"]]} {s["score"]:.2f}' for s in segments_info]
        xyxy = np.array([box[s['id']] for s in segments_info], dtype=np.float32)
        detections = sv.Detections(xyxy, confidence=np.array([s['score'] for s in segments_info]),
                                   class_id=np.array([s['category_id'] for s in segments_info]))
        blend = sv.BoundingBoxAnnotator().annotate(scene=blend, detections=detections)
        blend = sv.LabelAnnotator().annotate(scene=blend, detections=detections, labels=labels)

    if saver.dataset == 'gradio':
        saver.writer.write(blend[:, :, ::-1])
    elif saver.jpeg_encoder == 'device':  # an image finished on the host
        write(encode_jpeg_async(blend), _path(saver, saver.visualize_postfix, frame_name[:-4] + '.jpg'))
    else:
        _save(Image.fromarray(blend), saver, saver.visualize_postfix, frame_name[:-4] + '.jpg')


def _path(saver: ResultSaver, postfix: Optional[str], name: str) -> str:
    out = path.join(saver.output_root, postfix) if postfix is not None else saver.output_root
    if saver.video_name is not None:
        out = path.join(out, saver.video_name)
    os.makedirs(out, exist_ok=True)
    return path.join(out, name)


def _save(img: Image.Image, saver: ResultSaver, postfix: Optional[str], name: str):
    img.save(_path(saver, postfix, name))
