"""Times the evaluation criteria of dust3r_b200.losses on the GPU.

For both criteria of the reference's training recipes, on 32 pairs of 512x384 views whose ground truth comes from
synth_consistent_scene's cameras and depth maps (world points, camera poses, 25% of the pixels and a block per view invalid):
  - the CUDA path (csrc/criterion_ops.cu): ms per batch, and GB/s against the 29 B / pixel / view the criterion has to read
    at least (ground-truth points 12, mask 1, predicted points 12, confidence 4);
  - the host port's torch code (the reference's formulation) run directly on the same CUDA tensors;
  - the criterion's share of a loss_of_one_batch(..., symmetrize_batch=True) step of the flagship model (ViT-L / DPT 512,
    synthetic weights) on a batch of 16 pairs, which symmetrises to the same 32.
All times are CUDA-event times after warm-up.  Prints one JSON line, with the card's name and power limit read in the same run.

    python scripts/criterion_bench.py [--iters 20] [--warmup 3] [--out results/criterion_bench.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import dust3r_b200.losses as L  # noqa: E402
from dust3r_b200.inference import loss_of_one_batch  # noqa: E402
from dust3r_b200.utils.geometry import geotrf  # noqa: E402
from dust3r_b200.utils.synth import synth_consistent_scene  # noqa: E402
from common import card, events_ms  # noqa: E402

H, W = 384, 512
PAIRS = 32
TRAIN = "ConfLoss(Regr3D(L21, norm_mode='avg_dis'), alpha=0.2)"
TEST = "Regr3D_ScaleShiftInv(L21, gt_scale=True)"
BYTES_PER_PIXEL_VIEW = 29


def batch(n_pairs, device, seed=0):
    """(gt1, gt2, pred1, pred2) for n_pairs pairs of a consistent scene of 8 images."""
    edges = [(i, j) for i in range(8) for j in range(8) if i != j][:n_pairs]
    out, cams, _ = synth_consistent_scene(8, edges, H, W, seed=seed)
    g = torch.Generator().manual_seed(seed)
    i1 = torch.tensor([i for i, j in edges])
    i2 = torch.tensor([j for i, j in edges])
    p1, p2 = out['pred1']['pts3d'], out['pred2']['pts3d_in_other_view']

    def mask():
        m = torch.rand((n_pairs, H, W), generator=g) >= 0.25
        m[:, H // 4:H // 2, W // 4:W // 2] = False
        return m
    gt1 = dict(pts3d=geotrf(cams[i1], p1), valid_mask=mask(), camera_pose=cams[i1])
    gt2 = dict(pts3d=geotrf(cams[i1], p2), valid_mask=mask(), camera_pose=cams[i2])
    scale = 0.5 + torch.rand((n_pairs, 1, 1, 1), generator=g)
    pred1 = dict(pts3d=p1 * scale + 0.01 * torch.randn(p1.shape, generator=g), conf=out['pred1']['conf'])
    pred2 = dict(pts3d_in_other_view=p2 * scale + 0.01 * torch.randn(p2.shape, generator=g), conf=out['pred2']['conf'])
    return tuple({k: v.to(device) for k, v in d.items()} for d in (gt1, gt2, pred1, pred2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--skip-step', action='store_true', help='leave out the loss_of_one_batch step (no ViT-L model)')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('criterion_bench.py measures the GPU path and needs a CUDA H100')
    dev = torch.device('cuda', torch.cuda.current_device())
    inputs = batch(PAIRS, dev)
    floor_bytes = BYTES_PER_PIXEL_VIEW * 2 * PAIRS * H * W
    res = dict(card=card(dev), pairs=PAIRS, H=H, W=W, floor_bytes=floor_bytes, criteria={})
    for expr in (TRAIN, TEST):
        crit = eval(expr, vars(L))
        ours = events_ms(lambda: crit(*inputs), args.iters, args.warmup)
        with L.host_port():
            ref = events_ms(lambda: crit(*inputs), max(3, args.iters // 4), 1)
            ref_loss = float(crit(*inputs)[0])
        loss = float(crit(*inputs)[0])
        res['criteria'][expr] = dict(cuda_ms=round(ours, 4), host_port_on_gpu_ms=round(ref, 3), speedup=round(ref / ours, 2),
                                     cuda_GBps_vs_floor=round(floor_bytes / ours / 1e6, 1), loss=loss, host_port_loss=ref_loss)
    if not args.skip_step:
        sys.path.insert(0, ROOT)
        from bench import build_model
        net, _ = build_model(dev)
        half = PAIRS // 2
        gt1, gt2, _, _ = batch(half, dev, seed=1)
        g = torch.Generator().manual_seed(2)
        imgs = (torch.rand((2 * half, 3, H, W), generator=g) * 2 - 1).to(dev)
        views = [dict(gt, img=imgs[k * half:(k + 1) * half], true_shape=torch.tensor([[H, W]] * half),
                      instance=[str(k * half + i) for i in range(half)], idx=list(range(k * half, (k + 1) * half)))
                 for k, gt in enumerate((gt1, gt2))]
        for expr in (TRAIN, TEST):
            crit = eval(expr, vars(L))

            def step(c=crit):
                with torch.no_grad():
                    return loss_of_one_batch(tuple(dict(v) for v in views), net, c, dev, symmetrize_batch=True, ret='loss')
            with_ms = events_ms(step, max(3, args.iters // 4), 2)
            without_ms = events_ms(lambda: step(None), max(3, args.iters // 4), 1)
            r = res['criteria'][expr]
            r['step_ms'] = round(with_ms, 2)
            r['step_without_criterion_ms'] = round(without_ms, 2)
            r['share_of_step'] = round(r['cuda_ms'] / with_ms, 5)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
