"""Device PNG decode (csrc/png_decode.cu, deva/utils/png_decode.py) against Pillow on a host thread pool.

Reports, for ellipse id maps written by Pillow (480p P, 720p RGB, 1080p RGB) and by this project's device encoder:
  * the kernel time per file from CUDA events with the streams resident on the device, for one file alone and per file
    of a 25-file batch;
  * the time from file bytes on the host to decoded tensors on the device for a 25-frame batch (decode_results), next
    to the 16-thread Pillow decode plus pinned upload of the same files (png_pipeline.Decoder + Uploader);
  * the bytes each path uploads.
Prints one JSON line with the card and its power limit read in the same run."""
import argparse
import io
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402,F401  (puts the package on sys.path)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

import png_decode_cases as pdc  # noqa: E402
from bench_ingest import card  # noqa: E402

SHAPES = {'480p_P': ('P', 480, 854), '720p_RGB': ('RGB', 720, 1280), '1080p_RGB': ('RGB', 1080, 1920)}
FRAMES = 25


def files(mode, h, w, writer):
    """FRAMES ellipse id maps (a different seed per frame) as PNG bytes."""
    from deva.utils.png_encode import encode_png
    out = []
    for t in range(FRAMES):
        img = pdc.image('ellipse', mode, h, w, seed=t)
        if writer == 'pillow':
            out.append(pdc.pillow(img, mode))
        else:
            palette = [(37 * i + 11) % 256 for i in range(768)] if mode == 'P' else None
            out.append(encode_png(torch.from_numpy(img).cuda(), mode, palette))
    return out


def resident(datas):
    """Device arguments of one png_decode launch over datas (what decode_batch stages)."""
    from deva import _native as nat
    from deva.utils import png_decode as pd
    hds = [pd.parse(d) for d in datas]
    assert all(hds)
    streams = [hd.stream(d) for d, hd in zip(datas, hds)]
    desc = np.zeros((len(datas), nat.PNG_DESC_FIELDS), np.int64)
    s_at = o_at = w_at = 0
    for k, (hd, s) in enumerate(zip(hds, streams)):
        desc[k] = (s_at, len(s), hd.h, hd.w, hd.colour_type, hd.bits, o_at, w_at)
        s_at, o_at = s_at + len(s), o_at + (hd.nbytes + 15) // 16 * 16
        w_at += nat.png_decode_workspace_bytes(hd.h, hd.w, hd.colour_type, hd.bits)
    dev = torch.from_numpy(np.frombuffer(b''.join(streams), np.uint8).copy()).cuda()
    return (dev, torch.from_numpy(desc).cuda(), torch.empty(o_at, dtype=torch.uint8, device='cuda'),
            torch.empty(w_at, dtype=torch.uint8, device='cuda'),
            torch.empty(len(datas), dtype=torch.int32, device='cuda')), s_at + desc.nbytes


def kernel_ms(args, reps):
    from deva import _native as nat
    nat.png_decode(*args)
    torch.cuda.synchronize()
    assert not args[4].any(), args[4]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        nat.png_decode(*args)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def end_to_end(datas, paths, reps):
    """(device ms, Pillow + upload ms) for the batch, best of reps, alternating; and whether the results are equal."""
    from deva.utils import png_decode as pd
    from deva.utils.png_pipeline import Decoder, Uploader

    def read(p):
        return np.asarray(Image.open(p))
    dec, up = Decoder(read, 16), Uploader(torch.device('cuda'))
    dev_t, pil_t = [], []
    try:
        for _ in range(reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got = pd.decode_results(datas)
            torch.cuda.synchronize()
            dev_t.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            want = [up(a) for a in dec.frames(paths)]
            torch.cuda.synchronize()
            pil_t.append(time.perf_counter() - t0)
    finally:
        dec.close()
    equal = all(torch.equal(a, b) for a, b in zip(got, want))
    return min(dev_t) * 1e3, min(pil_t) * 1e3, equal


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    from deva import _native as nat
    nat.require_device()
    out = {'card': card(), 'cpu_threads': os.cpu_count(), 'frames_per_batch': FRAMES}
    with tempfile.TemporaryDirectory() as root:
        for writer in ('pillow', 'device_encoder'):
            for name, (mode, h, w) in SHAPES.items():
                datas = files(mode, h, w, writer)
                paths = []
                for t, d in enumerate(datas):
                    paths.append(os.path.join(root, f'{writer}_{name}_{t}.png'))
                    with open(paths[-1], 'wb') as f:
                        f.write(d)
                one, _ = resident(datas[:1])
                batch, up_bytes = resident(datas)
                dev_ms, pil_ms, equal = end_to_end(datas, paths, max(3, args.reps // 4))
                raw = sum(np.asarray(Image.open(io.BytesIO(d))).nbytes for d in datas)
                out[f'{writer}_{name}'] = {
                    'kernel_ms_one_file': round(kernel_ms(one, args.reps), 3),
                    'kernel_ms_per_file_in_batch': round(kernel_ms(batch, args.reps) / FRAMES, 3),
                    'batch_bytes_to_tensors_ms': {'device': round(dev_ms, 2), 'pillow_16_threads_and_upload':
                                                  round(pil_ms, 2)},
                    'uploaded_bytes': {'device': up_bytes, 'pillow': raw},
                    'file_kb_mean': round(sum(map(len, datas)) / len(datas) / 1024, 1), 'results_equal': equal}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
