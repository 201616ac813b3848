"""Two-GPU test of the product multi-GPU path (`-m gpu`; skipped on a single-GPU box): inference_sharded() over NCCL -- every
rank runs its slice of the pair list through the forward, ONE all_gather_into_tensor rebuilds the full result on every
rank (device resident), and it must equal single-GPU inference() of the whole list."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    from dust3r_b200.distributed import inference_sharded
    from dust3r_b200.inference import inference
    from dust3r_b200.image_pairs import make_pairs
    from dust3r_b200.utils.synth import synth_images
    from test_forward_gpu import _build, _small_cfgs
    cfg, H, W = _small_cfgs()['small_dpt']
    net, _ = _build(cfg, 11, dev)
    imgs = synth_images(4, H, W, seed=5)
    pairs = make_pairs(imgs, symmetrize=True)[:11]         # 11 pairs over 2 ranks: ragged split (6 + 5)
    out = inference_sharded(pairs, net, dev, batch_size=4, verbose=False, gather_device=dev)
    assert out['pred1']['pts3d'].device == dev and out['pred1']['pts3d'].shape[0] == len(pairs)
    ok = True
    if rank == 0:
        ref = inference(pairs, net, dev, batch_size=4, verbose=False, keep_on_device=True)
        for which, key in (('pred1', 'pts3d'), ('pred1', 'conf'), ('pred2', 'pts3d_in_other_view'), ('pred2', 'conf')):
            a, b = out[which][key], ref[which][key]
            err = float((a - b).abs().max() / b.abs().max())
            ok = ok and a.shape == b.shape and err < 1e-5
        ok = ok and out['view1']['idx'] == ref['view1']['idx'] and out['view2']['idx'] == ref['view2']['idx']
    # both ranks hold the same gathered tensors
    chk = out['pred2']['conf'].double().sum().reshape(1).clone()
    lst = [torch.zeros_like(chk) for _ in range(world)]
    dist.all_gather(lst, chk)
    ok = ok and bool(lst[0] == lst[1])
    q.put((rank, bool(ok)))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(900)
def test_inference_sharded_two_gpus_equals_single_gpu():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    world = 2
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert all(ok for _, ok in got), got


@pytest.mark.timeout(900)
def test_two_devices_driven_by_one_process():
    """One process, two GPUs, current device left at cuda:0: the forward and the aligner on cuda:1 must use cuda:1's stream, set
    their function attributes there too (they are per device) and give the bits cuda:0 gives."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    from test_forward_gpu import _build, _small_cfgs
    from dust3r_b200.utils.synth import synth_images, synth_pair_predictions
    from dust3r_b200.cloud_opt import global_aligner
    cfg, H, W = _small_cfgs()['small_dpt']
    imgs = synth_images(2, H, W, seed=5)
    res, losses = [], []
    n = 3
    edges = [(i, j) for i in range(n) for j in range(n) if i != j]
    out = synth_pair_predictions(n, edges, 32, 48, seed=0)
    torch.cuda.set_device(0)
    for d in (0, 1):
        dev = torch.device('cuda', d)
        net, _ = _build(cfg, 11, dev)
        r1, r2 = net(dict(img=imgs[0]['img'].to(dev), instance=['0']), dict(img=imgs[1]['img'].to(dev), instance=['1']))
        res.append((r1['pts3d'].cpu(), r2['conf'].cpu()))
        torch.manual_seed(0)
        scene = global_aligner(out, dev, verbose=False)
        scene.compute_global_alignment(init=None, niter=20)
        losses.append(scene.last_losses.cpu())
        assert torch.cuda.current_device() == 0
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    assert torch.equal(losses[0], losses[1]) and bool(torch.isfinite(losses[1]).all())
