"""Cost of the differentiable objective (d3r_align_loss_grad behind net() + loss.backward()) against the fused loop.

For BASELINE config 3 (8 views -> 28 pairs at 512x384, PointCloudOptimizer) and the config-5 graph (50 views -> 1225 pairs,
ModularPointCloudOptimizer, at --c5-hw pixels) it prints one JSON line each with
  grad_launch_us      CUDA-event time of one gradient launch (library profiler tag `align_grad`)
  fused_iter_us       CUDA-event time per iteration of compute_global_alignment (tag `align_stream` / `align_iter`)
  forward_backward_ms wall time per `loss = net(); loss.backward()` (host synchronised)
  adam_iter_ms        wall time per iteration of the reference loop body driven by torch.optim.Adam(betas=(0.9, 0.9))
together with the card line (GPU name, power limit and SM clocks) in `gpu` and the power limit alone in `power_limit`.

Usage:  python scripts/align_grad_bench.py [--iters 50] [--c5-hw 192 256]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dust3r_b200 import _lib  # noqa: E402
from dust3r_b200.cloud_opt import GlobalAlignerMode, global_aligner  # noqa: E402
from dust3r_b200.cloud_opt.commons import cosine_schedule  # noqa: E402
from dust3r_b200.utils.synth import synth_pair_predictions  # noqa: E402
from common import card, wall_ms  # noqa: E402


def per_launch_us(report, tag):
    r = report.get(tag)
    return None if not r else 1e3 * r['ms'] / r['count']


def bench(name, n, hw, mode, iters, dev):
    H, W = hw
    edges = [(i, j) for i in range(n) for j in range(i)]
    out = synth_pair_predictions(n, edges, H, W, seed=0)
    torch.manual_seed(0)
    net = global_aligner(out, dev, mode=mode, verbose=False)
    eng = net._get_engine()
    net.compute_global_alignment(init=None, niter=5)            # warm-up of both launch paths
    (net()).backward()
    torch.cuda.synchronize()

    _lib.prof_enable(True)                                      # clears earlier records
    net.compute_global_alignment(init=None, niter=iters)
    for _ in range(iters):
        eng.loss_and_grad()
    torch.cuda.synchronize()
    rep = _lib.prof_report()
    _lib.prof_enable(False)
    fused_tag = 'align_stream' if eng.kernel == 'stream' else 'align_iter'
    fused = rep[fused_tag]['ms'] * 1e3 / iters

    def fwd_bwd():
        net.zero_grad(set_to_none=True)
        net().backward()

    params = [p for p in net.parameters() if p.requires_grad]
    opt = torch.optim.Adam(params, lr=0.01, betas=(0.9, 0.9))
    it = [0]

    def adam_iter():
        for g in opt.param_groups:
            g['lr'] = cosine_schedule(it[0] / iters, 0.01, 1e-6)
        opt.zero_grad()
        loss = net()
        loss.backward()
        opt.step()
        it[0] += 1
    res = dict(config=name, n=n, E=len(edges), H=H, W=W, kernel=eng.kernel, grad_launch_us=per_launch_us(rep, 'align_grad'),
               fused_iter_us=fused, forward_backward_ms=wall_ms(fwd_bwd, iters, 1), adam_iter_ms=wall_ms(adam_iter, iters, 1))
    del net, eng, opt
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--c5-hw', type=int, nargs=2, default=(192, 256))
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    gpu = card(dev)
    runs = [('config3', 8, (384, 512), GlobalAlignerMode.PointCloudOptimizer),
            ('config5_graph', 50, tuple(a.c5_hw), GlobalAlignerMode.ModularPointCloudOptimizer)]
    for name, n, hw, mode in runs:
        r = bench(name, n, hw, mode, a.iters, dev)
        r.update(gpu=gpu, power_limit=gpu.split(', ')[1])
        print(json.dumps(r), flush=True)


if __name__ == '__main__':
    main()
