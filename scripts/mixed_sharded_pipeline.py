"""A phone-style scene of portrait and landscape shots end to end on the sharded path: 50 synthetic views, 25 at 512x384 and
25 at 384x512, complete symmetrised graph (2450 pairs of four size combinations), random-init ViT-L / DPT weights;
inference_sharded(keep='all' and keep='owned'), each followed by global_aligner_sharded (ModularPointCloudOptimizer,
init=None, cosine schedule), one process per GPU:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29515 \\
        scripts/mixed_sharded_pipeline.py [--niter 300] [--out results.json]

Prints one JSON line per keep mode from rank 0, with every rank's figures: its peak device memory
(torch.cuda.max_memory_allocated, reset before the forward), the forward + collective time, the alignment iterations/s and
the final loss; the card, its power limit and clocks are read in the same run.  Random-init weights: the numbers are timings
and memory, not a reconstruction."""
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


def views():
    """N views, landscape and portrait alternating, so that the first pairs of the list cover every size combination."""
    out = []
    for k in range(N):
        hw = (H, W) if k % 2 == 0 else (W, H)
        out.append(dict(synth_images(1, *hw, seed=21 + k)[0], idx=k, instance=str(k)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--niter', type=int, default=300)
    ap.add_argument('--batch-size', type=int, default=32)
    ap.add_argument('--out', default=None, help='also write the results to this JSON file')
    args = ap.parse_args()

    rank, world, local = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1)), int(os.environ.get('LOCAL_RANK', 0))
    dev = torch.device('cuda', local)
    torch.cuda.set_device(dev)
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ.setdefault('MASTER_PORT', '29515')
    dist.init_process_group('nccl', device_id=dev, rank=rank, world_size=world)

    net, _ = build_model(dev)
    pairs = make_pairs(views(), scene_graph='complete', prefilter=None, symmetrize=True)
    results = []
    for keep in ('all', 'owned'):
        # warm-up: every size combination, full batches, the communicator
        inference_sharded(pairs[:args.batch_size * world], net, dev, batch_size=args.batch_size, verbose=False, gather_device=dev,
                          return_images=False, keep=keep)
        barrier_sync()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
        t0 = time.perf_counter()
        fwd = inference_sharded(pairs, net, dev, batch_size=args.batch_size, verbose=False, gather_device=dev,
                                return_images=False, keep=keep)
        barrier_sync()
        t_fwd = time.perf_counter() - t0
        peak_fwd = torch.cuda.max_memory_allocated(dev)
        torch.manual_seed(0)
        scene = global_aligner_sharded(fwd, dev, mode=GlobalAlignerMode.ModularPointCloudOptimizer, verbose=False)
        scene.compute_global_alignment(init=None, niter=5)        # engine build, packing, module loads
        barrier_sync()
        t1 = time.perf_counter()
        loss = scene.compute_global_alignment(init=None, niter=args.niter, schedule='cosine', lr=0.01)
        barrier_sync()
        t_align = time.perf_counter() - t1
        mine = dict(rank=rank, peak_forward_bytes=peak_fwd, peak_bytes=torch.cuda.max_memory_allocated(dev))
        every = [None] * world
        dist.all_gather_object(every, mine)
        res = dict(keep=keep, world=world, n_views=N, n_pairs=len(pairs), sizes=f'{N // 2} x {W}x{H} + {N // 2} x {H}x{W}',
                   niter=args.niter, forward_and_collective_s=round(t_fwd, 3), pairs_per_s=round(len(pairs) / t_fwd, 1),
                   align_it_per_s=round(args.niter / t_align, 1), final_loss=loss, ranks=every, card=card(dev),
                   note='random-init weights; forward_and_collective_s is the forward plus the all-gather (all) or '
                        'all_to_all (owned); peaks include the model and the inputs')
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
