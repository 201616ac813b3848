"""Cost of the evaluation view stage (dust3r_b200.views: crop, resize, ImgNorm, unprojection of RGB-D frames) on the GPU and on
a host core, and its share of an evaluation step.

A batch is 16 items of two synthetic RGB-D frames (synth_rgbd_frame) at 512x384, i.e. 32 views, for two frame sizes: 12 Mpx
(4032x3024) and 1.4 Mpx (1440x960).  Per size:
  kernel_ms        CUDA-event time of the one d3r_prepare_views call of the batch (its three launches), frames resident in HBM
  call_ms          wall time of prepare_batch(device=cuda) from frames in HBM, host plan included, ending in a synchronise
  views_per_s      32 / call_ms
  floor_bytes      bytes the stage has to move at least: every RGB pixel of the principal-point crops once (3 B; the resize
                   reads them all), the depth pixels the nearest-neighbour resize samples (4 B per output pixel) and 29 B
                   written per output pixel (12 image, 4 depth, 12 points, 1 mask)
  GBps_vs_floor    floor_bytes / kernel_ms; divide by 3350 for the share of the H100 SXM's HBM3 data-sheet bandwidth
  host_ms_per_view prepare_views(device='cpu') -- Pillow, OpenCV and numpy, the reference's algorithm -- on ONE host core
                   (torch and OpenCV limited to one thread), ms per view, over a few views
and, for the 12 Mpx frames, step_ms = loss_of_one_batch(batch, flagship model (ViT-L / DPT 512, synthetic weights),
ConfLoss(Regr3D(L21, norm_mode='avg_dis'), alpha=0.2), symmetrize_batch=True) and share_of_step = call_ms / (call_ms + step_ms).
Prints one JSON line with the card's name and power limit and the host's core count, read in the same run.

    python scripts/views_bench.py [--iters 10] [--warmup 2] [--host-views 4] [--skip-step] [--out results/views_bench.json]
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dust3r_b200 import _lib, views  # noqa: E402
from dust3r_b200.utils.image import device_lut  # noqa: E402
from dust3r_b200.utils.synth import synth_rgbd_frame  # noqa: E402
from common import card, events_ms, wall_ms  # noqa: E402

RES = (512, 384)
ITEMS = 16
SIZES = {'12Mpx': (3024, 4032), '1.4Mpx': (960, 1440)}
OUT_BYTES_PER_PIXEL = 29
TRAIN = "ConfLoss(Regr3D(L21, norm_mode='avg_dis'), alpha=0.2)"


def frames_for(H, W, dev):
    """ITEMS items of two frames; two distinct frames shared by all items (their synthesis is slow at 12 Mpx)."""
    base = [synth_rgbd_frame(H, W, seed) for seed in (1, 2)]
    on_dev = [dict(f, img=torch.from_numpy(f['img']).to(dev), depthmap=torch.from_numpy(f['depthmap']).to(dev)) for f in base]
    return base, [(i, [dict(f, dataset='synth', label=str(i), instance=f'{i}_{v}') for v, f in enumerate(on_dev)])
                  for i in range(ITEMS)]


def floor_bytes(items):
    plans = [p for _, frames in items for p in views._plan_item(frames, RES, np.random.default_rng(0), False)]
    src = sum((p['crop1'][2] - p['crop1'][0]) * (p['crop1'][3] - p['crop1'][1]) * 3 for p in plans)
    return src + (4 + OUT_BYTES_PER_PIXEL) * RES[0] * RES[1] * len(plans)


def kernel_ms(items, dev, iters, warmup):
    """CUDA-event time of the d3r_prepare_views call alone, descriptors built once."""
    frames = [f for _, fr in items for f in fr]
    plans = [p for _, fr in items for p in views._plan_item(fr, RES, np.random.default_rng(0), False)]
    outs = [views._empty_outputs(p, dev) for p in plans]
    descs, keep = views.view_descriptors(frames, plans, outs, dev)
    desc_dev = torch.empty((len(frames) * ctypes.sizeof(_lib.ViewDesc),), dtype=torch.uint8, device=dev)
    lut = device_lut(dev)
    return events_ms(lambda: _lib.launch(dev, 'd3r_prepare_views', len(frames), descs, desc_dev.data_ptr(), lut.data_ptr()),
                     iters, warmup)


def host_ms_per_view(base, n):
    import cv2
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    cv2.setNumThreads(1)
    try:
        rng = np.random.default_rng(0)
        views.prepare_views(base, RES, rng=rng, device='cpu')
        t0 = time.perf_counter()
        done = 0
        while done < n:
            done += len(views.prepare_views(base, RES, rng=rng, device='cpu'))
        return 1e3 * (time.perf_counter() - t0) / done
    finally:
        torch.set_num_threads(threads)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--host-views', type=int, default=4)
    ap.add_argument('--skip-step', action='store_true', help='leave out the loss_of_one_batch step (no ViT-L model)')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('views_bench.py measures the GPU path and needs a CUDA H100')
    dev = torch.device('cuda', torch.cuda.current_device())
    res = dict(card=card(dev), host_cores=os.cpu_count(), host_cores_usable=len(os.sched_getaffinity(0)), resolution=RES,
               views_per_batch=2 * ITEMS, sizes={})
    step_items = None
    for name, (H, W) in SIZES.items():
        base, items = frames_for(H, W, dev)
        k_ms = kernel_ms(items, dev, args.iters, args.warmup)
        call = wall_ms(lambda: views.prepare_batch(items, RES, seed=1, device=dev), args.iters, args.warmup)
        fb = floor_bytes(items)
        res['sizes'][name] = dict(frame=[W, H], kernel_ms=round(k_ms, 4), call_ms=round(call, 3),
                                  views_per_s=round(2 * ITEMS / call * 1e3, 1), floor_bytes=fb,
                                  GBps_vs_floor=round(fb / k_ms / 1e6, 1),
                                  host_ms_per_view=round(host_ms_per_view(base, args.host_views), 2))
        if name == '12Mpx':
            step_items = items
    if not args.skip_step:
        import dust3r_b200.losses as L
        from dust3r_b200.inference import loss_of_one_batch
        from bench import build_model
        net, _ = build_model(dev)
        crit = eval(TRAIN, vars(L))
        batch = views.prepare_batch(step_items, RES, seed=1, device=dev)

        def step():
            with torch.no_grad():
                return loss_of_one_batch(tuple(dict(v) for v in batch), net, crit, dev, symmetrize_batch=True, ret='loss')
        step_ms = events_ms(step, max(3, args.iters // 2), 2)
        call = res['sizes']['12Mpx']['call_ms']
        res.update(step_ms=round(step_ms, 2), share_of_step=round(call / (call + step_ms), 4))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
