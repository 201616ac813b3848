"""Cost of decoding PNG photographs on the GPU (`decode_png`, csrc/png_ops.cu) and of `load_images(device=cuda)` end to end.

Seeded photograph-like images are encoded here by Pillow at its default compression level, at 4032x3024 (12 Mpx) and at
1280x960.  The script prints one JSON line with, per size (keys suffixed _12mp / _1mp):
  file_bytes            size of one file
  kernel_ms             CUDA-event time of one d3r_png_decode call (every kernel of it) from the zlib stream already in HBM,
                        mean over --iters
  MBps                  compressed bytes / kernel time
  load_gpu_ms           wall time of load_images(folder of --n such files, size=512, device=cuda): files read, chunks walked
                        and CRC-checked by the worker threads, zlib streams uploaded, decode + resize on the GPU
  load_host_decode_ms   the same call with every file decoded by Pillow on the worker threads (the path taken before the
                        GPU decoder existed; pixels uploaded, resize on the GPU)
  load_cpu_ms           load_images(device=None): the reference's host pipeline
  pillow_ms_per_file    one Pillow decode (exif_transpose + convert('RGB')) on one host core
  same_bits             the three load_images results are equal
together with the card line (GPU name, power limit and SM clocks) in `gpu`, read in the same run.

Usage:  python scripts/png_bench.py [--n 50] [--iters 10] [--out FILE]
"""
import argparse
import contextlib
import ctypes
import io
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dust3r_b200 import _lib  # noqa: E402
from dust3r_b200.utils import image as image_mod  # noqa: E402
from dust3r_b200.utils import png  # noqa: E402
from common import card, events_ms  # noqa: E402


def photo(h, w, seed):
    """Smooth colour fields, edges and sensor-like noise: compresses like a photograph."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.stack([128 + 90 * np.sin(x / (60 + 17 * c) + y / (45 + 11 * c) + seed) for c in range(3)], axis=-1)
    img += rng.normal(0, 6, img.shape).astype(np.float32)
    img[((x // 97 + y // 83) % 4 == 0)] *= 0.7
    return np.clip(img, 0, 255).astype(np.uint8)


def encode(arr):
    import PIL.Image
    buf = io.BytesIO()
    PIL.Image.fromarray(arr).save(buf, 'PNG')
    return buf.getvalue()


def kernel_ms(data, dev, iters):
    head = png.parse(data)
    desc = png.descriptor(head, png.orientation(head))
    lib = _lib.get_lib()
    n = len(head['idat'])
    ws_bytes = int(lib.d3r_png_decode_workspace_bytes(ctypes.byref(desc), n))
    src = torch.frombuffer(bytearray(head['idat']), dtype=torch.uint8).to(dev)
    out = torch.empty((desc.height, desc.width, 3), dtype=torch.uint8, device=dev)
    status = torch.empty((1,), dtype=torch.int32, device=dev)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)

    def call():
        _lib.launch(dev, 'd3r_png_decode', ctypes.byref(desc), src.data_ptr(), n, out.data_ptr(), status.data_ptr(), ws.data_ptr(),
                    ws_bytes)
    ms = events_ms(call, iters, 2)
    assert int(status.item()) == 0
    assert np.array_equal(out.cpu().numpy(), image_mod._pillow_rgb(data))
    return ms


def load_ms(folder, device, host_decode=False):
    from dust3r_b200.utils.image import load_images
    stage = image_mod._png_stage
    if host_decode:
        image_mod._png_stage = lambda data: None
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            load_images(folder, size=512, device=device)        # warm-up: module load, tables, pinned allocator
            if device is not None:
                torch.cuda.synchronize()
            t0 = time.perf_counter()
            views = load_images(folder, size=512, device=device)
            if device is not None:
                torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0), views
    finally:
        image_mod._png_stage = stage


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=50)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    _lib.require_cuda_device(dev)
    r = dict(n=args.n)
    for tag, (H, W) in (('12mp', (3024, 4032)), ('1mp', (960, 1280))):
        files = [encode(photo(H, W, s)) for s in range(3)]
        r[f'file_bytes_{tag}'] = len(files[0])
        r[f'kernel_ms_{tag}'] = kernel_ms(files[0], dev, args.iters)
        r[f'MBps_{tag}'] = len(files[0]) / r[f'kernel_ms_{tag}'] / 1e3
        t0 = time.perf_counter()
        image_mod._pillow_rgb(files[0])
        r[f'pillow_ms_per_file_{tag}'] = 1e3 * (time.perf_counter() - t0)
        with tempfile.TemporaryDirectory() as folder:
            for i in range(args.n):
                with open(os.path.join(folder, f'{i:03d}.png'), 'wb') as f:
                    f.write(files[i % len(files)])
            r[f'load_gpu_ms_{tag}'], gpu_views = load_ms(folder, dev)
            r[f'load_host_decode_ms_{tag}'], hd_views = load_ms(folder, dev, host_decode=True)
            r[f'load_cpu_ms_{tag}'], cpu_views = load_ms(folder, None)
            r[f'same_bits_{tag}'] = all(torch.equal(a['img'].cpu(), b['img'].cpu()) and torch.equal(a['img'].cpu(), c['img'])
                                        for a, b, c in zip(gpu_views, hd_views, cpu_views))
    gpu = card(dev)
    r.update(gpu=gpu, power_limit=gpu.split(', ')[1] if ', ' in gpu else 'unknown')
    line = json.dumps(r)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
