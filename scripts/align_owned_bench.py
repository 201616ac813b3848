"""inference_sharded(keep='all') against inference_sharded(keep='owned'), each followed by global_aligner_sharded, on the
config-5 graph (50 views -> 1225 pairs, 512x384, ModularPointCloudOptimizer, init=None, cosine schedule), one process per
GPU:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29513 \\
        scripts/align_owned_bench.py [--niter 300] [--backend nccl|gloo] [--out results.json]

Prints one JSON line per keep mode from rank 0, with every rank's figures: the bytes of predictions it keeps, its peak
device memory (torch.cuda.max_memory_allocated, reset before the forward, and the same above the memory the model and the
inputs already held), the forward + routing time, the alignment iterations/s and the final loss; the card, its power limit
and clocks are read in the same run.  --backend gloo runs every rank on GPU 0 (routing through host memory): its memory
figures are valid, its times are not.  Random-init weights: the numbers are timings and memory, not a reconstruction."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

from bench import build_model
from common import barrier_sync, card
from dust3r_b200.cloud_opt import GlobalAlignerMode
from dust3r_b200.distributed import global_aligner_sharded, inference_sharded
from dust3r_b200.image_pairs import make_pairs
from dust3r_b200.utils.synth import synth_images

H, W, N = 384, 512, 50


def kept_bytes(out):
    n = 0
    for which in ('pred1', 'pred2'):
        for v in out[which].values():
            n += sum(t.numel() * t.element_size() for t in (v if isinstance(v, list) else [v]) if t is not None)
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--niter', type=int, default=300)
    ap.add_argument('--backend', default='nccl', choices=('nccl', 'gloo'))
    ap.add_argument('--batch-size', type=int, default=32)
    ap.add_argument('--out', default=None, help='also write the results to this JSON file')
    args = ap.parse_args()

    rank, world, local = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1)), int(os.environ.get('LOCAL_RANK', 0))
    dev = torch.device('cuda', local if args.backend == 'nccl' else 0)
    torch.cuda.set_device(dev)
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ.setdefault('MASTER_PORT', '29513')
    if args.backend == 'nccl':
        dist.init_process_group('nccl', device_id=dev, rank=rank, world_size=world)
    else:
        dist.init_process_group('gloo', rank=rank, world_size=world)

    net, _ = build_model(dev)
    imgs = synth_images(N, H, W, seed=21)
    pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=False)
    results = []
    for keep in ('all', 'owned'):
        # warm-up with full batches: the forward's work buffers then count as resident in both legs
        inference_sharded(pairs[:args.batch_size * world], net, dev, batch_size=args.batch_size, verbose=False, gather_device=dev,
                          return_images=False, keep=keep)
        barrier_sync()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
        resident = torch.cuda.memory_allocated(dev)
        t0 = time.perf_counter()
        fwd = inference_sharded(pairs, net, dev, batch_size=args.batch_size, verbose=False, gather_device=dev,
                                return_images=False, keep=keep)
        barrier_sync()
        t_fwd = time.perf_counter() - t0
        torch.manual_seed(0)
        scene = global_aligner_sharded(fwd, dev, mode=GlobalAlignerMode.ModularPointCloudOptimizer, verbose=False)
        scene.compute_global_alignment(init=None, niter=5)        # engine build, packing, module loads
        barrier_sync()
        t1 = time.perf_counter()
        loss = scene.compute_global_alignment(init=None, niter=args.niter, schedule='cosine', lr=0.01)
        barrier_sync()
        t_align = time.perf_counter() - t1
        peak = torch.cuda.max_memory_allocated(dev)
        mine = dict(rank=rank, kept_bytes=kept_bytes(fwd), peak_bytes=peak, peak_above_resident_bytes=peak - resident,
                    routing_buffers=fwd['owned'].allocated if keep == 'owned' else None)
        every = [None] * world
        dist.all_gather_object(every, mine)
        res = dict(keep=keep, world=world, backend=args.backend, n_views=N, n_pairs=len(pairs), size=f'{W}x{H}', niter=args.niter,
                   forward_and_route_s=round(t_fwd, 3) if args.backend == 'nccl' else 'not measured',
                   align_it_per_s=round(args.niter / t_align, 1) if args.backend == 'nccl' else 'not measured',
                   final_loss=loss, ranks=every, card=card(dev),
                   note='random-init weights; forward_and_route_s is the forward plus the all-gather (all) or all_to_all (owned)')
        if rank == 0:
            print(json.dumps(res), flush=True)
            results.append(res)
        del scene, fwd
        torch.cuda.empty_cache()
        barrier_sync()

    if rank == 0 and args.out:
        with open(args.out, 'w') as f:
            json.dump(results, f, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
