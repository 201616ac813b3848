"""Cost of decoding JPEG photographs on the GPU (`decode_jpeg`, csrc/jpeg_ops.cu) and of `load_images(device=cuda)` end to end.

Seeded 4032x3024 (12 Mpx) photographs are encoded here by Pillow at quality 90, 4:2:0, without and with restart markers (one per
MCU row).  The script prints one JSON line with
  kernel_ms / kernel_ms_rst     CUDA-event time of one d3r_jpeg_decode call (every kernel of it) from bytes already in HBM,
                                mean over --iters
  MBps / MBps_rst               compressed bytes / kernel time
  file_bytes / file_bytes_rst   size of the files
  load_gpu_ms                   wall time of load_images(folder of --n such files, size=512, device=cuda): files read and
                                headers parsed by the worker threads, compressed bytes uploaded, decode + resize on the GPU
  load_host_decode_ms           the same call with every file decoded by Pillow on the worker threads (the path taken before
                                the GPU decoder existed; pixels uploaded, resize on the GPU)
  load_cpu_ms                   load_images(device=None): the reference's host pipeline
  same_bits                     the three load_images results are equal
together with the card line (GPU name, power limit and SM clocks) in `gpu` and the power limit alone in `power_limit`, read
in the same run.

Usage:  python scripts/jpeg_bench.py [--n 50] [--iters 20] [--out FILE]
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
from dust3r_b200.utils import jpeg  # noqa: E402
from common import card, events_ms  # noqa: E402


def photo(h, w, seed):
    """Smooth colour fields, edges and sensor-like noise: compresses like a photograph (about 2 bits per pixel at q90)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.stack([128 + 90 * np.sin(x / (60 + 17 * c) + y / (45 + 11 * c) + seed) for c in range(3)], axis=-1)
    img += rng.normal(0, 6, img.shape).astype(np.float32)
    img[((x // 97 + y // 83) % 4 == 0)] *= 0.7
    return np.clip(img, 0, 255).astype(np.uint8)


def encode(arr, **kw):
    import PIL.Image
    buf = io.BytesIO()
    PIL.Image.fromarray(arr).save(buf, 'JPEG', quality=90, subsampling=2, **kw)
    return buf.getvalue()


def kernel_ms(data, dev, iters):
    desc = jpeg.descriptor(jpeg.parse(data), jpeg.orientation(data))
    lib = _lib.get_lib()
    n = len(data)
    ws_bytes = int(lib.d3r_jpeg_decode_workspace_bytes(ctypes.byref(desc), n))
    src = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(dev)
    out = torch.empty((desc.height, desc.width, 3), dtype=torch.uint8, device=dev)
    status = torch.empty((1,), dtype=torch.int32, device=dev)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)

    def call():
        _lib.launch(dev, 'd3r_jpeg_decode', ctypes.byref(desc), src.data_ptr(), n, out.data_ptr(), status.data_ptr(), ws.data_ptr(),
                    ws_bytes)
    ms = events_ms(call, iters, 3)
    assert int(status.item()) == 0
    assert np.array_equal(out.cpu().numpy(), image_mod._pillow_rgb(data))
    return ms


def load_ms(folder, device, host_decode=False):
    from dust3r_b200.utils.image import load_images
    stage = image_mod._jpeg_stage
    if host_decode:
        image_mod._jpeg_stage = lambda data: None
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
        image_mod._jpeg_stage = stage


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=50)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    _lib.require_cuda_device(dev)
    H, W = 3024, 4032
    arrs = [photo(H, W, s) for s in range(5)]
    plain = encode(arrs[0])
    rst = encode(arrs[0], restart_marker_rows=1)
    r = dict(n=args.n, hw=[H, W], file_bytes=len(plain), file_bytes_rst=len(rst))
    r['kernel_ms'] = kernel_ms(plain, dev, args.iters)
    r['kernel_ms_rst'] = kernel_ms(rst, dev, args.iters)
    r['MBps'] = len(plain) / r['kernel_ms'] / 1e3
    r['MBps_rst'] = len(rst) / r['kernel_ms_rst'] / 1e3
    with tempfile.TemporaryDirectory() as folder:
        files = [encode(a) for a in arrs]
        for i in range(args.n):
            with open(os.path.join(folder, f'{i:03d}.jpg'), 'wb') as f:
                f.write(files[i % len(files)])
        r['load_gpu_ms'], gpu_views = load_ms(folder, dev)
        r['load_host_decode_ms'], hd_views = load_ms(folder, dev, host_decode=True)
        r['load_cpu_ms'], cpu_views = load_ms(folder, None)
        r['same_bits'] = all(torch.equal(a['img'].cpu(), b['img'].cpu()) and torch.equal(a['img'].cpu(), c['img'])
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
