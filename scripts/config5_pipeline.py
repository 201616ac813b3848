"""BASELINE configs[4] end to end: 50 synthetic views -> 1225 pairs at 512x384, forward sharded over the ranks of one box
(torchrun, one process per GPU), ONE NCCL all-gather of the pointmaps (inference_sharded -> PairOutputGather), then
global_aligner(ModularPointCloudOptimizer) for 300 iterations on rank 0's GPU (alignment = replicas only).  Prints one JSON line
with the seconds of every stage.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29511 scripts/config5_pipeline.py [n_views]
"""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

from bench import build_model, H, W
from common import barrier_sync, card
from dust3r_b200.distributed import inference_sharded
from dust3r_b200.image_pairs import make_pairs
from dust3r_b200.cloud_opt import global_aligner, GlobalAlignerMode
from dust3r_b200.utils.synth import synth_images


def main():
    n_views = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    rank, world, local = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1)), int(os.environ.get('LOCAL_RANK', 0))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    net, cfg = build_model(dev)
    imgs = synth_images(n_views, H, W, seed=21)
    for im in imgs:
        im['img'] = im['img'].pin_memory()
    pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=False)
    assert len(pairs) == n_views * (n_views - 1) // 2

    # warm-up (weight repack, lazy module loads, NCCL communicator)
    inference_sharded(pairs[:2 * world], net, dev, batch_size=32, verbose=False, gather_device=dev)
    barrier_sync()
    t0 = time.perf_counter()
    out = inference_sharded(pairs, net, dev, batch_size=32, verbose=False, gather_device=dev, return_images=False)
    barrier_sync()
    t_fwd = time.perf_counter() - t0
    res = dict(n_views=n_views, n_pairs=len(pairs), world=world, forward_and_gather_s=round(t_fwd, 3), pairs_per_s=round(len(pairs) / t_fwd, 1))
    if rank == 0:
        t0 = time.perf_counter()
        torch.manual_seed(0)
        scene = global_aligner(out, dev, mode=GlobalAlignerMode.ModularPointCloudOptimizer, verbose=False)
        torch.cuda.synchronize()
        t_build = time.perf_counter() - t0
        t0 = time.perf_counter()
        loss = scene.compute_global_alignment(init=None, niter=300, schedule='cosine', lr=0.01)
        torch.cuda.synchronize()
        t_align = time.perf_counter() - t0
        res.update(aligner_build_s=round(t_build, 3), align_300_iters_s=round(t_align, 3), iters_per_s=round(300 / t_align, 1), final_loss=loss,
                   total_s=round(t_fwd + t_build + t_align, 3), mem_GB=round(torch.cuda.max_memory_allocated() / 1e9, 1),
                   card=card(dev), note='random-init weights: the pointmaps are not a consistent scene; init=None (no MST) -- timing only')
        print(json.dumps(res), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
