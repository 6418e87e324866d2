"""``DeviceLoader``: a reader's items with the frames and masks decoded, resized and normalised on the device.

It replaces a driver's ``DataLoader(reader, batch_size=1, num_workers=2)`` line; the rest of the loop runs unchanged.
Item ``i`` is ``default_collate([reader[i]])`` (what ``DataLoader(reader, batch_size=1)`` yields) except that
``data['rgb']`` and ``data['mask']`` are CUDA tensors on the current device, produced there: rgb bit for bit at the
frame's own size and within 1e-6 when resized; masks, soft masks, ``valid_labels`` and every info field exactly equal.

With the demos' ``SimpleVideoReader`` it replaces ``DataLoader(reader, batch_size=None, collate_fn=no_collate,
num_workers=8)``: item ``i`` is ``(frame, im_path)`` where ``frame`` is the CUDA uint8 [H, W, 3] tensor equal to
``torch.from_numpy(reader[i][0])``, neither collated nor normalised (the demos' processors hand the raw frame to the
detectors and the overlay, and normalise it themselves through ``demo_utils.get_input_frame_for_deva``).

Pipeline, for windows of ``prefetch // 2`` frames (at most ``prefetch`` frames are read ahead):
  * host threads run each frame's ``reader.plan(i)``, read its files and parse them (``jpeg_decode.parse``,
    ``png_decode.parse``; a ``size_dir`` shape is read from the file's header, without a decode);
  * on a loader-owned stream, the window's JPEG frames go to one ``jpeg_decode`` launch and its mask PNGs to one
    ``png_decode`` launch, followed by the resizes (``frame_from_rgb8``, ``mask_from_index8``, ``mask_ids_from_u8``,
    ``soft_from_u8``);
  * the decode statuses and, per ID-mask frame, a 256-bin histogram of the resized mask (its ``valid_labels``: one
    small download per ID-mask frame, i.e. the first frame, or every annotated frame with ``use_all_masks``) are
    copied to pinned memory and read once, when the window's first frame is handed out.  The next window is enqueued
    before that, so in steady state the read finds the copy complete; there is no per-frame host synchronisation;
  * the consumer's current stream waits on the window's event, and handed-out tensors are ``record_stream``ed.

The device covers JPEG frames that ``jpeg_decode.parse`` accepts; ``VideoReader`` ID masks from P or L PNGs; soft
masks from L PNGs (all three layouts); ``DetectionVideoReader`` masks from P, L or RGB PNGs.  Every other frame -
a declined or corrupt file, an RGBA / 16-bit / interlaced mask, ``segmentation_from_dict`` - is ``reader[i]`` on the
host, collated and uploaded, so it equals the reader by construction, errors included (same type and message at the
same index).  Items are handed out in order and reader state (``DetectionVideoReader.is_rgb``) evolves as in a
sequential pass.
"""
import os
from concurrent.futures import ThreadPoolExecutor
from os import path
from typing import List, NamedTuple, Optional

import torch
from torch.utils.data import default_collate

from deva.inference import frame_io
from deva.inference.data.detection_video_reader import DetectionVideoReader
from deva.inference.data.simple_video_reader import SimpleVideoReader
from deva.inference.data.video_reader import (MASK_DETECTION, MASK_ID, MASK_SOFT, MASK_SOFT_MULTI, Plan,
                                              VideoReader)
from deva.utils import device_decode, jpeg_decode, png_decode


class _Parsed(NamedTuple):
    """A frame the device reads: its plan, the frame's JPEG, its shape and its mask PNGs (bytes and headers)."""
    plan: Plan
    image: tuple          # (bytes, jpeg_decode.Header)
    shape: tuple          # (h, w) reported in info['shape']
    masks: List[tuple]    # [(bytes, png_decode.Header)]; empty without a mask


def _header_shape(data) -> Optional[tuple]:
    hd = jpeg_decode.parse(data) or png_decode.parse(data)
    return None if hd is None else (hd.h, hd.w)


def _parse(reader, i) -> Optional[_Parsed]:
    """Item ``i``'s files read and parsed when the device can read them all, else None (the host reads the item)."""
    try:
        plan = reader.plan(i)
        data = device_decode.read_bytes(plan.image)
        hd = None if data is None else jpeg_decode.parse(data)
        if hd is None:
            return None
        shape = (hd.h, hd.w)
        if plan.size_path is not None:
            size_data = device_decode.read_bytes(plan.size_path)
            shape = None if size_data is None else _header_shape(size_data)
            if shape is None:
                return None
        masks = []
        if plan.mask_kind in (MASK_ID, MASK_DETECTION) and not path.exists(plan.masks[0]):
            pass  # an optional mask that is absent: no mask
        elif plan.mask_kind in (MASK_ID, MASK_DETECTION, MASK_SOFT, MASK_SOFT_MULTI):
            modes = {MASK_ID: ('P', 'L'), MASK_DETECTION: ('P', 'L', 'RGB')}.get(plan.mask_kind, ('L',))
            for p in plan.masks:
                m = device_decode.read_bytes(p)
                mh = None if m is None else png_decode.parse(m)
                if mh is None or mh.mode not in modes:
                    return None
                masks.append((m, mh))
            if len({(mh.h, mh.w) for _, mh in masks}) != 1:
                return None
        elif plan.mask_kind is not None:
            return None
        return _Parsed(plan, (data, hd), shape, masks)
    except Exception:  # noqa: BLE001  (the host path reads the item and raises the reader's own error)
        return None


class _Window:
    """One window's device work: per frame its outputs, and the pinned copy of the statuses read at hand-out."""

    def __init__(self, start, parsed, size, stream):
        """size: the reader's working short side (< 0: the frame's own size; None: the raw uint8 frame)."""
        self.start, self.parsed = start, parsed
        self.out = [None] * len(parsed)
        self.keep = []
        on = [k for k, p in enumerate(parsed) if p is not None]
        with torch.cuda.stream(stream):
            statuses, self.status_of = [], {}
            if on:
                st, frames, keep = jpeg_decode.enqueue([parsed[k].image[1] for k in on])
                statuses.append(st)
                self.keep.append(keep)
            files = [(k, f) for k in on for f in parsed[k].masks]
            masks = []
            if files:
                st, masks, keep = png_decode.enqueue([f for _, f in files])
                statuses.append(st)
                self.keep.append(keep)
            for j, k in enumerate(on):
                self.status_of[k] = [j]
            for j, (k, _) in enumerate(files):
                self.status_of[k].append(len(on) + j)
            hists = []
            size_arg = None if size is None or size < 0 else size
            for j, k in enumerate(on):
                p = parsed[k]
                rgb = frames[j] if size is None else frame_io.frame_from_rgb8(frames[j], size=size_arg, resize='reader')
                mine = [masks[m] for m, (kk, _) in enumerate(files) if kk == k]
                mask, hist = None, None
                if mine and p.plan.mask_kind == MASK_ID:
                    mask = frame_io.mask_from_index8(mine[0], size_arg)
                    hist = len(hists)
                    hists.append(torch.bincount(mask.view(-1), minlength=256))
                elif mine and p.plan.mask_kind == MASK_DETECTION:
                    mask = frame_io.mask_ids_from_u8(mine[0], size_arg)
                elif mine:
                    mask = frame_io.soft_from_u8(torch.stack(mine), size_arg)
                self.out[k] = (rgb, mask, hist)
            self.status = torch.empty(len(on) + len(files), dtype=torch.int32, pin_memory=True)
            if statuses:
                self.status.copy_(torch.cat(statuses), non_blocking=True)
            self.hist = torch.empty(len(hists), 256, dtype=torch.int64, pin_memory=True)
            if hists:
                self.hist.copy_(torch.stack(hists), non_blocking=True)
            self.ready = torch.cuda.Event()
            self.ready.record(stream)
        self.read = False

    def device_ok(self, k) -> bool:
        """Whether frame k of the window was read on the device (reads the statuses once: synchronises with the
        window's copy, already complete in steady state)."""
        if self.parsed[k] is None:
            return False
        if not self.read:
            self.ready.synchronize()
            self.read = True
        return all(int(self.status[j]) == 0 for j in self.status_of[k])


class DeviceLoader:
    """Iterates ``reader`` (this package's ``VideoReader`` or ``DetectionVideoReader``) like
    ``DataLoader(reader, batch_size=1)``, or a ``SimpleVideoReader`` like ``DataLoader(reader, batch_size=None,
    collate_fn=no_collate)``, with the frames and masks read on the device (see the module's docstring).
    prefetch: frames read ahead of the one handed out; num_threads: host threads reading and parsing files (default:
    the host's cores, at most 8).  ``host_indices`` lists the items of the last pass the host read."""

    def __init__(self, reader, *, prefetch: int = 16, num_threads: Optional[int] = None):
        if not isinstance(reader, (VideoReader, DetectionVideoReader, SimpleVideoReader)):
            raise TypeError(f'DeviceLoader reads a deva.inference.data VideoReader, DetectionVideoReader or '
                            f'SimpleVideoReader, not {type(reader).__name__}')
        if prefetch < 1:
            raise ValueError(f'DeviceLoader: prefetch must be at least 1, got {prefetch}')
        self.reader = reader
        self.raw = isinstance(reader, SimpleVideoReader)
        self.window = max(1, prefetch // 2)
        self.num_threads = num_threads or min(8, os.cpu_count() or 1)
        self.host_indices: List[int] = []

    def __len__(self):
        return len(self.reader)

    def _host_item(self, i):
        dev = torch.device('cuda', torch.cuda.current_device())
        if self.raw:
            frame, im_path = self.reader[i]
            return torch.from_numpy(frame).to(dev), im_path
        data = default_collate([self.reader[i]])
        for key in ('rgb', 'mask'):
            if key in data:
                data[key] = data[key].to(dev)
        return data

    def _device_item(self, win, k):
        p = win.parsed[k]
        rgb, mask, hist = win.out[k]
        if self.raw:
            consumer = torch.cuda.current_stream()
            consumer.wait_event(win.ready)
            rgb.record_stream(consumer)
            return rgb, p.plan.image
        if p.plan.mask_kind == MASK_DETECTION:
            item = self.reader.assemble(p.plan, None, p.shape, mask, p.masks[0][1].mode == 'RGB' if p.masks else None)
        else:
            labels = None
            if mask is not None:
                labels = torch.arange(1, mask.shape[0] + 1) if p.plan.mask_kind != MASK_ID else \
                    torch.nonzero(win.hist[hist][1:]).view(-1) + 1
            item = self.reader.assemble(p.plan, None, p.shape, mask, labels)
        consumer = torch.cuda.current_stream()
        consumer.wait_event(win.ready)
        out = {}
        for key, v in item.items():
            if key in ('rgb', 'mask'):
                t = rgb if key == 'rgb' else mask
                t.record_stream(consumer)
                out[key] = t.unsqueeze(0)
            else:
                out[key] = default_collate([v])
        return out

    def __iter__(self):
        n = len(self.reader)
        self.host_indices = []
        stream = torch.cuda.Stream()
        stream.wait_stream(torch.cuda.current_stream())
        starts = list(range(0, n, self.window))
        with ThreadPoolExecutor(self.num_threads) as pool:
            def submit(s):
                return [pool.submit(_parse, self.reader, i) for i in range(s, min(n, s + self.window))]

            def enqueue(s, futures):
                return _Window(s, [f.result() for f in futures], None if self.raw else self.reader.size, stream)

            futures = {s: submit(s) for s in starts[:2]}
            pending = enqueue(starts[0], futures.pop(starts[0])) if starts else None
            for w, s in enumerate(starts):
                win = pending
                if w + 2 < len(starts):
                    futures[starts[w + 2]] = submit(starts[w + 2])
                pending = enqueue(starts[w + 1], futures.pop(starts[w + 1])) if w + 1 < len(starts) else None
                for k in range(len(win.parsed)):
                    if win.device_ok(k):
                        yield self._device_item(win, k)
                    else:
                        self.host_indices.append(s + k)
                        yield self._host_item(s + k)
