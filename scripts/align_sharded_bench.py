"""Sharded global alignment (distributed.global_aligner_sharded) against the fused single-GPU loop, on BASELINE configs 5
(50 views -> 1225 pairs, ModularPointCloudOptimizer) and 3 (8 views -> 28 pairs, PointCloudOptimizer), 512x384, 300
iterations, cosine schedule, one process per GPU:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29512 \\
        scripts/align_sharded_bench.py [--niter 300] [--configs 5,3] [--no-e2e] [--out results.json]

Prints one JSON line per config from rank 0: iterations/s of the fused loop on rank 0's GPU alone and of the sharded loop
at world N; the per-iteration split of the sharded loop into pixel pass, all-reduce and small step (CUDA events, in a run
of its own); the packed observation bytes of every rank and the max / mean ratio; and, for config 5, the end to end time of
inference_sharded + sharded alignment.  At N = 1 the sharded loop is the split iteration with a one-rank all-reduce: what
the split costs against the fused launch.

The gradient leg (--grad-iters, 0 skips it): host-synchronised wall ms per `loss = scene(); loss.backward()` on the fused
scene on rank 0's GPU alone (one d3r_align_loss_grad launch) and on the sharded scene at world N (sharded_loss_and_grad), and,
in a run of its own, the CUDA-event split of the sharded call into gradient pixel pass, all-reduce, gradient small step and
the log-depth-gradient broadcasts.  The card, its power limit and clocks are read in the same run."""
import argparse
import ctypes
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

from bench import build_model
from common import barrier_sync, card, wall_ms
from dust3r_b200 import _lib
from dust3r_b200.cloud_opt import GlobalAlignerMode, global_aligner
from dust3r_b200.distributed import _AlignShard, global_aligner_sharded, inference_sharded, shard_images
from dust3r_b200.image_pairs import make_pairs
from dust3r_b200.utils.synth import synth_images, synth_pair_predictions

H, W = 384, 512
CONFIGS = {'5': (50, 'ModularPointCloudOptimizer'), '3': (8, 'PointCloudOptimizer')}


def sharded_scene(out, mode, dev, world):
    """The scene global_aligner_sharded returns, also at world 1 (where global_aligner_sharded hands back the fused scene)."""
    torch.manual_seed(0)
    scene = global_aligner(out, dev, mode=GlobalAlignerMode[mode], verbose=False)
    deg = [0] * scene.n_imgs
    for i, j in scene.edges:
        deg[i] += 1
        deg[j] += 1
    scene._align_shard = _AlignShard(shard_images(scene.imshapes, deg, world), None)
    return scene


def timed_alignment(scene, niter):
    scene.compute_global_alignment(init=None, niter=5)          # warm-up: engine build, packing, module loads
    barrier_sync()
    t0 = time.perf_counter()
    loss = scene.compute_global_alignment(init=None, niter=niter, schedule='cosine', lr=0.01)
    barrier_sync()
    return time.perf_counter() - t0, loss


def split_breakdown(eng, niter):
    """Mean ms of the pixel pass, the all-reduce and the small step per iteration (CUDA events around each)."""
    eng.reset_adam()
    eng.sched = torch.from_numpy(eng.make_schedule(niter, 0.01, 'cosine', 1e-6)).to(eng.device)
    eng.loss_out = torch.zeros((niter,), dtype=torch.float32, device=eng.device)
    eng._sync_start()
    eng.prepare()
    d = eng._desc()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(niter)]
    barrier_sync()
    for it in range(niter):
        ev[it][0].record()
        if eng.n_items:
            _lib.launch(eng.device, 'd3r_align_pixel_pass', ctypes.byref(d), it)
        ev[it][1].record()
        dist.all_reduce(eng._reduce, op=dist.ReduceOp.SUM)
        ev[it][2].record()
        _lib.launch(eng.device, 'd3r_align_small_step', ctypes.byref(d), it)
        ev[it][3].record()
    barrier_sync()
    parts = [sum(ev[it][k].elapsed_time(ev[it][k + 1]) for it in range(niter)) / niter for k in range(3)]
    return dict(pixel_pass_ms=round(parts[0], 4), all_reduce_ms=round(parts[1], 4), small_step_ms=round(parts[2], 4))


def fwd_bwd(scene):
    scene.zero_grad(set_to_none=True)
    scene().backward()


def timed_ms(fn, iters):
    """Wall ms per call of the collective `fn` on every rank: host clock between two barriers after device synchronises."""
    fn()
    barrier_sync()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    barrier_sync()
    return 1e3 * (time.perf_counter() - t0) / iters


def grad_breakdown(eng, iters):
    """Mean ms of the gradient pixel pass, the all-reduce, the gradient small step and the log-depth-gradient broadcasts of
    one sharded_loss_and_grad (CUDA events around each, the same launches and collectives in the same order)."""
    with torch.cuda.device(eng.device):
        eng._sync_start()
        eng.prepare()
    d = eng._desc()
    loss = torch.zeros((), dtype=torch.float32, device=eng.device)
    d.loss_out = loss.data_ptr()
    logd_grad = torch.zeros_like(eng.logd)
    small_grad = torch.empty((eng.n_small,), dtype=torch.float32, device=eng.device)
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(5)] for _ in range(iters)]
    barrier_sync()
    for it in range(iters):
        ev[it][0].record()
        if eng.n_items:
            _lib.launch(eng.device, 'd3r_align_grad_pixel_pass', ctypes.byref(d), logd_grad.data_ptr())
        ev[it][1].record()
        dist.all_reduce(eng._reduce, op=dist.ReduceOp.SUM)
        ev[it][2].record()
        _lib.launch(eng.device, 'd3r_align_grad_small_step', ctypes.byref(d), small_grad.data_ptr(), None)
        ev[it][3].record()
        eng._sync_end(logd_grad)
        ev[it][4].record()
    barrier_sync()
    parts = [sum(ev[it][k].elapsed_time(ev[it][k + 1]) for it in range(iters)) / iters for k in range(4)]
    return dict(grad_pixel_pass_ms=round(parts[0], 4), grad_all_reduce_ms=round(parts[1], 4),
                grad_small_step_ms=round(parts[2], 4), grad_broadcasts_ms=round(parts[3], 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--niter', type=int, default=300)
    ap.add_argument('--no-e2e', action='store_true')
    ap.add_argument('--configs', default='5,3')
    ap.add_argument('--grad-iters', type=int, default=20, help='calls per timing of the gradient leg (0: no gradient leg)')
    ap.add_argument('--out', default=None, help='also write the results of every config to this JSON file')
    args = ap.parse_args()

    rank, world, local = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1)), int(os.environ.get('LOCAL_RANK', 0))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ.setdefault('MASTER_PORT', '29512')
    dist.init_process_group('nccl', device_id=dev, rank=rank, world_size=world)

    res_all = []
    for key in args.configs.split(','):
        n, mode = CONFIGS[key]
        edges = [(i, j) for i in range(n) for j in range(i)]
        out = synth_pair_predictions(n, edges, H, W, seed=0)
        res = dict(config=key, n_views=n, n_pairs=len(edges), mode=mode, niter=args.niter, world=world, card=card(dev))
        # fused single-GPU loop on rank 0's GPU alone
        if rank == 0:
            torch.manual_seed(0)
            scene = global_aligner(out, dev, mode=GlobalAlignerMode[mode], verbose=False)
            scene.compute_global_alignment(init=None, niter=5)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            loss = scene.compute_global_alignment(init=None, niter=args.niter, schedule='cosine', lr=0.01)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            res.update(fused_1gpu_s=round(dt, 4), fused_1gpu_it_per_s=round(args.niter / dt, 1), fused_final_loss=loss)
            if args.grad_iters:
                res.update(grad_fused_1gpu_ms=round(wall_ms(lambda: fwd_bwd(scene), args.grad_iters, 2), 4))
            del scene
            torch.cuda.empty_cache()
        barrier_sync()
        scene = sharded_scene(out, mode, dev, world)
        dt, loss = timed_alignment(scene, args.niter)
        eng = scene._get_engine()
        obs = [None] * world
        dist.all_gather_object(obs, (eng.owned, eng.total_obs * 16))
        res.update(sharded_s=round(dt, 4), sharded_it_per_s=round(args.niter / dt, 1), sharded_final_loss=loss,
                   shards=[o[0] for o in obs], obs_bytes_per_rank=[o[1] for o in obs],
                   obs_bytes_max_over_mean=round(max(o[1] for o in obs) / (sum(o[1] for o in obs) / world), 4))
        res.update(split_breakdown(eng, args.niter))
        if args.grad_iters:
            fwd_bwd(scene)
            res.update(grad_sharded_ms=round(timed_ms(lambda: fwd_bwd(scene), args.grad_iters), 4))
            res.update(grad_breakdown(eng, args.grad_iters))
        del scene, eng
        torch.cuda.empty_cache()
        if key == '5' and not args.no_e2e:
            # config 5 end to end: sharded forward + one all-gather, then the sharded alignment on every rank
            net, _ = build_model(dev)
            imgs = synth_images(n, H, W, seed=21)
            pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=False)
            inference_sharded(pairs[:2 * world], net, dev, batch_size=32, verbose=False, gather_device=dev)   # warm-up
            barrier_sync()
            t0 = time.perf_counter()
            fwd = inference_sharded(pairs, net, dev, batch_size=32, verbose=False, gather_device=dev, return_images=False)
            barrier_sync()
            t_fwd = time.perf_counter() - t0
            del net
            torch.manual_seed(0)
            scene = sharded_scene(fwd, mode, dev, world) if world == 1 else global_aligner_sharded(
                fwd, dev, mode=GlobalAlignerMode[mode], verbose=False)
            barrier_sync()
            t_build = time.perf_counter() - t0 - t_fwd
            t1 = time.perf_counter()
            scene.compute_global_alignment(init=None, niter=args.niter, schedule='cosine', lr=0.01)
            barrier_sync()
            t_align = time.perf_counter() - t1
            res.update(e2e_forward_and_gather_s=round(t_fwd, 3), e2e_aligner_build_s=round(t_build, 3),
                       e2e_align_s=round(t_align, 3), e2e_total_s=round(time.perf_counter() - t0, 3),
                       e2e_note='random-init weights, init=None: timing only; the align time includes the engine build and packing')
            del scene, fwd
            torch.cuda.empty_cache()
        if rank == 0:
            print(json.dumps(res), flush=True)
            res_all.append(res)
        barrier_sync()

    if rank == 0 and args.out:
        with open(args.out, 'w') as f:
            json.dump(res_all, f, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
