"""Cost of localising a query on the GPU: run_pnp on CUDA tensors (csrc/pnp_ops.cu + the host SQPnP refinement) against the
reference's cv2.solvePnPRansac path, and one localize() of a query against 20 map views.

PnP problems: 100 000 synthetic correspondences (oracle/pnp_float64.synth_problem, 0.5 px noise) at 95 / 50 / 20 % inliers,
the run_pnp settings (SOLVEPNP_SQPNP, 10 000 iterations, confidence 0.9999, 5 px).  Per ratio the JSON line holds
  gpu_wall_ms        run_pnp(CUDA tensors) wall time, host clock around the call (it ends in a device synchronise)
  gpu_kernel_ms      CUDA-event time of the loop alone (pnp_ransac: every kernel of d3r_pnp_ransac)
  hypotheses         hypotheses the GPU loop evaluated
  gpu_inliers        inliers of its winning hypothesis
  cv2_wall_ms        run_pnp(numpy), i.e. cv2.solvePnPRansac on the host (cv2.getNumThreads() threads)
  cv2_inliers        solvePnPRansac's inlier count
  rot_err_deg, trans_err  the GPU pose against the ground truth
localize: a 512x384 query and 20 map views with the full-size synthetic model (vitl_512_dpt, random weights, so the matches
are not meaningful geometry): wall time of one localize() call, and its correspondence count.  The card line (name, power
limit, SM clocks) is read in the same run.

Usage:  python scripts/pnp_bench.py [--iters 5] [--skip-localize] [--out FILE]
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
from common import card, events_ms  # noqa: E402
from dust3r_b200.localization import localize, localize_matches, pnp_ransac, run_pnp  # noqa: E402
from oracle.pnp_float64 import synth_problem  # noqa: E402


def _median_ms(fn, iters):
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts))


def bench_pnp(dev, ratio, iters):
    import cv2
    p2, p3, K, R, t, _ = synth_problem(100_000, ratio, 0.5, seed=1)
    t2, t3 = torch.from_numpy(p2).to(dev), torch.from_numpy(p3).to(dev)
    run_pnp(t2, t3, K)
    torch.cuda.synchronize()
    gpu_wall = _median_ms(lambda: run_pnp(t2, t3, K), iters)
    kernel = events_ms(lambda: pnp_ransac(t2, t3, K), iters, 1)
    result, _, _ = pnp_ransac(t2, t3, K)
    ok, T = run_pnp(t2, t3, K)
    W = np.linalg.inv(T)
    cv_iters = 1 if ratio < 0.3 else iters
    cv_wall = _median_ms(lambda: run_pnp(p2, p3, K), cv_iters)
    _, _, _, inl = cv2.solvePnPRansac(p3, p2, K, None, flags=cv2.SOLVEPNP_SQPNP, iterationsCount=10_000, reprojectionError=5,
                                      confidence=0.9999)
    return dict(gpu_wall_ms=gpu_wall, gpu_kernel_ms=kernel, hypotheses=int(result[2]), gpu_inliers=int(result[1]),
                cv2_wall_ms=cv_wall, cv2_threads=cv2.getNumThreads(), cv2_inliers=0 if inl is None else len(inl),
                rot_err_deg=float(np.degrees(np.arccos(np.clip((np.trace(W[:3, :3].T @ R) - 1) / 2, -1, 1)))),
                trans_err=float(np.linalg.norm(W[:3, 3] - t)))


def bench_localize(dev, iters):
    import sys as _sys
    _sys.path.insert(0, ROOT)
    from bench import build_model
    from PIL import Image
    net, _ = build_model(dev)
    H, W, n_maps = 384, 512, 20
    g = torch.Generator().manual_seed(0)
    rgb = lambda: torch.rand((3, H, W), generator=g) * 2 - 1
    query = dict(rgb_rescaled=rgb(), to_orig=np.diag([2.0, 2.0, 1.0]), intrinsics=np.array([[800.0, 0, 512], [0, 800, 384], [0, 0, 1]]),
                 distortion=None, rgb=Image.new('RGB', (2 * W, 2 * H)))
    maps = [dict(rgb_rescaled=rgb(), valid_rescaled=torch.ones((H, W), dtype=torch.bool),
                 pts3d_rescaled=torch.randn((H, W, 3), generator=g)) for _ in range(n_maps)]
    localize(query, maps, net, dev, conf_thr=0.0, rng=random.Random(0))
    torch.cuda.synchronize()
    wall = _median_ms(lambda: localize(query, maps, net, dev, conf_thr=0.0, rng=random.Random(0)), iters)
    p2, _ = localize_matches(query, maps, net, dev, conf_thr=0.0)
    return dict(localize_wall_ms=wall, map_views=n_maps, size=f'{W}x{H}', correspondences=0 if p2 is None else len(p2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--skip-localize', action='store_true')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    res = dict(gpu=card(dev))
    for ratio in (0.95, 0.5, 0.2):
        res[f'pnp_{int(100 * ratio)}pct'] = bench_pnp(dev, ratio, a.iters)
    if not a.skip_localize:
        res['localize'] = bench_localize(dev, a.iters)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
