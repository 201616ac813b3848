"""Cost of sky segmentation (`segment_sky` / `scene.mask_sky()`) on the GPU against the host path.

For n images of HxW (default 50 at 384x512, the config-5 scene; synthetic sky over textured ground plus noise, seeded) it prints
one JSON line with
  kernel_ms          CUDA-event time of one d3r_segment_sky call for all n images (its seven kernels), mean over --iters
  kernel_GBps        algorithmic bytes / kernel_ms
  algo_bytes         compulsory traffic of the call: 44 B per pixel (csrc/sky_ops.cu kBytesPerPixel)
  mask_sky_ms        wall time of scene.mask_sky() on a device scene (PointCloudOptimizer, edges (i, i+1) both ways): the
                     scene's deepcopy, the pinned upload of scene.imgs, quantisation, the kernels and the im_conf writes
  segment_ms         wall time of the batched segmentation alone, from the float host images (pinned upload included)
  host_ms            wall time of the host path (OpenCV + scipy, dust3r_b200.viz.segment_sky on numpy) on the same images
together with the card line (GPU name, power limit and SM clocks) in `gpu` and the power limit alone in `power_limit`, read
in the same run.

Usage:  python scripts/sky_bench.py [--n 50] [--hw 384 512] [--iters 20] [--out FILE]
"""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dust3r_b200 import _lib  # noqa: E402
from dust3r_b200.cloud_opt import global_aligner  # noqa: E402
from dust3r_b200.cloud_opt.scene_ops import _quantise, segment_sky_host_images  # noqa: E402
from dust3r_b200.utils.synth import synth_pair_predictions, synth_sky_image  # noqa: E402
from dust3r_b200.viz import segment_sky  # noqa: E402
from common import card, events_ms, wall_ms  # noqa: E402

BYTES_PER_PIXEL = 44


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=50)
    ap.add_argument('--hw', type=int, nargs=2, default=(384, 512))
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    dev = torch.device('cuda')
    _lib.require_cuda_device(dev)
    lib = _lib.get_lib()
    n, (H, W) = a.n, a.hw
    images = [synth_sky_image(H, W, seed=k) for k in range(n)]

    # the kernels alone, on pre-quantised bytes: CUDA events around back-to-back calls
    total = n * H * W
    rgb = _quantise(torch.from_numpy(np.concatenate([x.reshape(-1) for x in images])).to(dev))
    hw = torch.tensor([[H, W]] * n, dtype=torch.int32, device=dev)
    off = torch.arange(n, dtype=torch.int64, device=dev) * (H * W)
    out = torch.empty((total,), dtype=torch.uint8, device=dev)
    ws = torch.empty((int(lib.d3r_segment_sky_workspace_bytes(n, total)),), dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream

    def kernels():
        _lib.check(lib.d3r_segment_sky(n, hw.data_ptr(), off.data_ptr(), H * W, total, rgb.data_ptr(), out.data_ptr(), ws.data_ptr(),
                                       ws.numel(), stream))
    kernel_ms = events_ms(kernels, a.iters, 3)

    segment_ms = wall_ms(lambda: segment_sky_host_images(images, dev), a.iters, 1)

    edges = [(i, i + 1) for i in range(n - 1)]
    out_pairs = synth_pair_predictions(n, edges + [(j, i) for i, j in edges], H, W, seed=1)
    for view in ('view1', 'view2'):
        out_pairs[view]['img'] = torch.stack([torch.from_numpy(2 * images[i] - 1).permute(2, 0, 1) for i in out_pairs[view]['idx']])
    scene = global_aligner(out_pairs, dev, verbose=False)
    mask_sky_ms = wall_ms(scene.mask_sky, max(a.iters // 4, 3), 1)

    host_iters = max(a.iters // 10, 1)
    t = time.perf_counter()
    for _ in range(host_iters):
        host = [segment_sky(x) for x in images]
    host_ms = 1e3 * (time.perf_counter() - t) / host_iters
    same = all(torch.equal(h, d.cpu()) for h, d in zip(host, segment_sky_host_images(images, dev)))

    gpu = card(dev)
    algo = BYTES_PER_PIXEL * total
    r = dict(bench='segment_sky', n=n, H=H, W=W, kernel_ms=round(kernel_ms, 4), kernel_GBps=round(algo / kernel_ms / 1e6, 1),
             algo_bytes=algo, segment_ms=round(segment_ms, 3), mask_sky_ms=round(mask_sky_ms, 3), host_ms=round(host_ms, 2),
             host_threads=int(__import__('cv2').getNumThreads()), sky_fraction=round(float(out.float().mean()), 4),
             host_equals_device=same, gpu=gpu, power_limit=gpu.split(', ')[1])
    line = json.dumps(r)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
