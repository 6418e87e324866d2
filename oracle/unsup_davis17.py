"""numpy restatement of the reference's unsupervised DAVIS 2017 post-processing (``limit_max_id``,
deva/inference/postprocess_unsup_davis17.py:11-56).

Per frame, one ``np.unique(return_counts=True)`` gives every label's area (the reference makes one full-frame pass per
label), and the rewrite is one table lookup (the reference makes one pass per list entry).  The rules it restates:
  1. videos and frames are every entry of sorted(os.listdir(...)); an output keeps its input's name;
  2. a 2-D frame's label is its value, a colour frame's R * 65536 + G * 256 + B; label 0 is ignored;
  3. the selection pass appends each frame's labels by (area, label) descending, only the first max - len(list) when they
     do not all fit, and stops after the frame that fills the list; no de-duplication; assert len(list) <= max;
  4. every frame is rewritten: a listed label takes its last position + 1, others 0; saved as a P PNG with the palette;
  5. input and output may be the same directory (a frame is read before it is written);
  6. a 256th entry raises numpy's OverflowError on the video's first rewrite, before any of its files is written;
  7. max = 0 writes all-zero masks; a negative max fails the assert.
Checked against the unmodified reference's outputs in tests/golden/unsup_davis17.{json,npz}.
"""
import os

import numpy as np
from PIL import Image


def frame_labels(file) -> np.ndarray:
    a = np.array(Image.open(file)).astype(np.int64)
    return a if a.ndim == 2 else a[:, :, 0] * 65536 + a[:, :, 1] * 256 + a[:, :, 2]


def limit_max_id(input_path, output_path, max_num_objects, palette):
    for video in sorted(os.listdir(input_path)):
        video_path = os.path.join(input_path, video)
        frames = sorted(os.listdir(video_path))
        existing = []
        for frame in frames:
            labels, areas = np.unique(frame_labels(os.path.join(video_path, frame)), return_counts=True)
            keep = labels != 0
            labels, areas = labels[keep], areas[keep]
            by_area = [int(v) for v in labels[np.lexsort((labels, areas))[::-1]]]
            room = max_num_objects - len(existing)
            existing += by_area if len(by_area) <= room else by_area[:room]
            if len(existing) == max_num_objects:
                break
        assert len(existing) <= max_num_objects
        last = {v: i + 1 for i, v in enumerate(existing)}  # a repeated label keeps its last position
        table = np.array(sorted(last), np.int64)
        index = np.array([last[v] for v in table.tolist()], np.int64)
        for frame in frames:
            mask = frame_labels(os.path.join(video_path, frame))
            if len(existing) > 255:
                raise OverflowError('Python integer 256 out of bounds for uint8')
            out = np.zeros(mask.shape, np.uint8)
            if len(table):
                i = np.minimum(np.searchsorted(table, mask), len(table) - 1)
                hit = table[i] == mask
                out[hit] = index[i[hit]]
            img = Image.fromarray(out)
            img.putpalette(palette)
            os.makedirs(os.path.join(output_path, video), exist_ok=True)
            img.save(os.path.join(output_path, video, frame))
