"""Unsupervised DAVIS 2017 post-processing (the reference's deva/inference/postprocess_unsup_davis17.py) with the pixel
work on the device.

``limit_max_id`` keeps at most ``max_num_objects`` objects per video and rewrites every frame as a palette PNG of their
1-based indices, as the reference does:
  * videos and frames are every entry of ``sorted(os.listdir(...))``; an output file keeps its input's name;
  * a P or L frame's label is its pixel value, an RGB(A) frame's is ``R * 65536 + G * 256 + B``; label 0 is background;
  * the selection pass walks the frames in order: a frame's labels sorted by (area, label) descending are appended to
    the list (only the first ``max_num_objects - len(list)`` of them when they do not all fit) and the pass stops after
    the frame that fills the list.  The list is not de-duplicated: a label seen in k frames takes k entries;
  * every frame is rewritten: a label in the list takes its last position + 1 (uint8), every other pixel 0.  A list of
    256 or more entries raises numpy's ``OverflowError`` before any file of its video is written.

Per video each file is decoded once on a pool of host threads and uploaded through pinned slots, and the frames stay on
the device for both passes.  ``deva_b200_label_areas`` counts every frame's labels, and the per-frame lists come to the
host once; the selection runs there, on lists of at most a few thousand entries.  The (label -> index) table goes back
to the device, ``deva_b200_label_to_index`` rewrites every frame, and the index maps come back through pinned memory
to be encoded on the thread pool.  With ``png_decoder='device'`` (or ``DEVA_B200_PNG_DECODER=device``) the files are
read on the pool and decoded a video at a time on the device (png_pipeline.DeviceDecoder); a file the device does not
take is read by read_frame as before.  With ``png_encoder='device'`` (or ``DEVA_B200_PNG_ENCODER=device``) they are encoded
as PNGs on the device instead (deva/utils/png_encode.py), and only the compressed files come back.  Files are read in
full before any of their video is written, so input_path == output_path (as evaluation/eval_with_detections.py calls
it) is safe.

Supported frames are P, L, RGB and RGBA uint8 images (everything the result saver writes); another mode raises
``ValueError`` naming the file, where the reference would read the frame.  Importing this module does not initialise
CUDA.
"""
import os
import sys
from os import path

import numpy as np
import torch
from PIL import Image

from deva.utils.device_download import write
from deva.utils.png_encode import encode_png_async, resolve_encoder
from deva.utils.png_decode import resolve_decoder
from deva.utils.png_pipeline import Decoder, DeviceDecoder, Uploader

CAPACITY = 1024  # label table entries per frame; a frame with more distinct labels is counted again with a larger table
MODES = ('P', 'L', 'RGB', 'RGBA')


class _Unreadable:
    """A file that could not be read as a frame: its error is raised where the reference would meet it."""

    def __init__(self, error):
        self.error = error


def read_frame(file):
    """uint8 [h, w] (P, L) or [h, w, 3 | 4] (RGB, RGBA) of one file, or an _Unreadable."""
    try:
        img = Image.open(file)
        if img.mode not in MODES:
            raise ValueError(f'{file}: image mode {img.mode} is not supported (expected one of {", ".join(MODES)})')
        return np.asarray(img)
    except Exception as e:  # noqa: BLE001  (raised later, in the reference's order)
        return _Unreadable(e)


def _save(mask: np.ndarray, palette, file: str):
    img = Image.fromarray(mask)
    img.putpalette(palette)
    img.save(file)


def _label_lists(frames, dev):
    """[(labels, areas)] of every device frame, as host int32 arrays."""
    from deva import _native
    pitch = 2 * CAPACITY + 2
    buf = torch.empty(len(frames), pitch, dtype=torch.int32, device=dev)
    for t, f in enumerate(frames):
        _native.label_areas(f, buf[t, :CAPACITY], buf[t, CAPACITY:2 * CAPACITY], buf[t, 2 * CAPACITY:])
    host = buf.cpu().numpy()
    lists = []
    for t, row in enumerate(host):
        n = int(row[2 * CAPACITY])
        if n >= 0:
            lists.append((row[:n], row[CAPACITY:CAPACITY + n]))
            continue
        # more than CAPACITY labels: a table of one entry per pixel cannot overflow
        cap = frames[t].shape[0] * frames[t].shape[1]
        labels, counts, state = (torch.empty(k, dtype=torch.int32, device=dev) for k in (cap, cap, 2))
        _native.label_areas(frames[t], labels, counts, state)
        lists.append(_native.label_areas_result(labels.cpu().numpy(), counts.cpu().numpy(), state.cpu().numpy()))
    return lists


def select_objects(lists, max_num_objects):
    """The reference's selection pass over the frames' (labels, areas): -> (list of labels, whether it stopped early)."""
    existing_objects = []
    for labels, areas in lists:
        order = np.lexsort((labels, areas))[::-1]  # area descending, then label descending
        labels_sorted_by_area = [int(v) for v in labels[order]]
        if len(labels_sorted_by_area) + len(existing_objects) <= max_num_objects:
            existing_objects += labels_sorted_by_area
        else:
            existing_objects += labels_sorted_by_area[:max_num_objects - len(existing_objects)]
        if len(existing_objects) == max_num_objects:
            return existing_objects, True
    return existing_objects, False


def index_table(existing_objects):
    """Sorted int32 labels and their int32 output indices: a label listed several times keeps its last position + 1."""
    last = {label: i + 1 for i, label in enumerate(existing_objects)}
    labels = np.array(sorted(last), np.int32)
    return labels, np.array([last[v] for v in labels.tolist()], np.int32)


def _limit_video(decoder, upload, video_path, out_dir, max_num_objects, palette, png_encoder):
    from deva import _native
    dev = upload.device
    frames = sorted(os.listdir(video_path))
    decoded, unreadable = [], None
    for a in decoder.frames([path.join(video_path, f) for f in frames]):
        if isinstance(a, _Unreadable):
            unreadable = a.error
            break
        decoded.append(a)
    on_dev = [upload(a) for a in decoded]

    existing_objects, stopped = select_objects(_label_lists(on_dev, dev), max_num_objects)
    if not stopped and unreadable is not None:
        raise unreadable  # the selection pass reads up to the unreadable file
    assert len(existing_objects) <= max_num_objects
    if frames and len(existing_objects) > 255:
        # the reference's first `new_mask[mask == label] = 256` on its uint8 mask: numpy's own error (or, under a numpy
        # that wraps instead, no error, and the kernel's (uint8) cast wraps the same way)
        np.zeros(1, np.uint8)[np.zeros(1, bool)] = 256
    if not decoded:
        return

    labels, index = index_table(existing_objects)
    labels, index = torch.from_numpy(labels).to(dev), torch.from_numpy(index).to(dev)
    starts = [0]  # 16-byte aligned slices of one buffer
    for f in on_dev:
        starts.append(starts[-1] + (f.shape[0] * f.shape[1] + 15) // 16 * 16)
    out = torch.empty(starts[-1], dtype=torch.uint8, device=dev)
    maps = [out[s:s + f.shape[0] * f.shape[1]].view(f.shape[0], f.shape[1]) for f, s in zip(on_dev, starts)]
    for f, m in zip(on_dev, maps):
        _native.label_to_index(f, labels, index, m)
    os.makedirs(out_dir, exist_ok=True)
    if png_encoder == 'device':
        pngs = [encode_png_async(m, 'P', palette) for m in maps]
        writes = [decoder.pool.submit(write, p, path.join(out_dir, name)) for p, name in zip(pngs, frames)]
    else:
        host = torch.empty(out.numel(), dtype=torch.uint8, pin_memory=True)
        host.copy_(out, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        host_np = host.numpy()
        writes = [decoder.pool.submit(_save, host_np[s:s + f.shape[0] * f.shape[1]].reshape(f.shape[0], f.shape[1]),
                                      palette, path.join(out_dir, name))
                  for f, s, name in zip(on_dev, starts, frames)]
    for w in writes:
        w.result()
    if unreadable is not None:
        raise unreadable  # the rewrite pass wrote the frames before it


def limit_max_id(input_path, output_path, max_num_objects=20, *, palette=None, num_threads=None, png_encoder=None,
                 png_decoder=None):
    """palette: the PNGs' palette; None = DAVIS's (deva.utils.palette.davis_palette, which comes from the reference
    checkout).  num_threads: host threads that decode and encode PNGs.  png_encoder: 'pil' or 'device'; None reads
    DEVA_B200_PNG_ENCODER (default 'pil').  png_decoder: 'pil' or 'device'; None reads DEVA_B200_PNG_DECODER (default
    'pil')."""
    png_encoder = resolve_encoder(png_encoder)
    png_decoder = resolve_decoder(png_decoder)
    if palette is None:
        from deva.utils.palette import davis_palette as palette
    from deva import _native
    _native.require_device()
    dev = torch.device('cuda', torch.cuda.current_device())
    decoder = DeviceDecoder(read_frame, dev, num_threads=num_threads) if png_decoder == 'device' else \
        Decoder(read_frame, num_threads)
    upload = Uploader(dev)
    try:
        for video in sorted(os.listdir(input_path)):
            _limit_video(decoder, upload, path.join(input_path, video), path.join(output_path, video), max_num_objects,
                         palette, png_encoder)
    finally:
        decoder.close()


if __name__ == '__main__':
    input_path = sys.argv[1]
    output_path = sys.argv[2]
    limit_max_id(input_path, output_path)
