"""world_size-2 gloo test of the pair sharding + all-gather plumbing (the forward itself needs an H100, so a
deterministic stand-in model produces the per-pair outputs)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT


class _FakeModel:
    """pred depends only on the pair's images -> results are comparable across shardings."""
    conf_mode = ('exp', 1, float('inf'))

    def __call__(self, view1, view2):
        a, b = view1['img'], view2['img']
        B, _, H, W = a.shape
        pts = (a[:, :3].permute(0, 2, 3, 1) + 2 * b[:, :3].permute(0, 2, 3, 1)).contiguous()
        conf = 1 + (a[:, 0] - b[:, 1]).abs()
        return dict(pts3d=pts, conf=conf), dict(pts3d_in_other_view=pts * 0.5, conf=conf + 1)


class _FakeModelNoConf(_FakeModel):
    conf_mode = None

    def __call__(self, view1, view2):
        r1, r2 = super().__call__(view1, view2)
        return dict(pts3d=r1['pts3d']), dict(pts3d_in_other_view=r2['pts3d_in_other_view'])


def _pairs(n_imgs):
    from dust3r_b200.image_pairs import make_pairs
    from dust3r_b200.utils.synth import synth_images
    imgs = synth_images(abs(n_imgs), 16, 32, seed=4)
    # n_imgs < 0: one-directional pairs (a single pair for 2 images -> rank 1 of 2 has no work)
    return make_pairs(imgs, symmetrize=n_imgs > 0)


def _worker(rank, world, port, n_imgs, q, conf=True):
    sys.path.insert(0, ROOT)
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from dust3r_b200.distributed import inference_sharded, shard_bounds
    pairs = _pairs(n_imgs)
    out = inference_sharded(pairs, _FakeModel() if conf else _FakeModelNoConf(), 'cpu', batch_size=2, verbose=False)
    assert ('conf' in out['pred1']) == conf and ('conf' in out['pred2']) == conf
    q.put((rank, out['view1']['idx'], out['view2']['idx'], out['pred1']['pts3d'].numpy(),
           out['pred2']['conf'].numpy() if conf else out['pred2']['pts3d_in_other_view'].numpy()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('n_imgs,conf', [(3, True), (4, True), (-2, True), (-3, True), (3, False)])
def test_sharded_inference_equals_single_process(n_imgs, conf):
    """even split (4 images -> 12 pairs), ragged split (3 -> 6 pairs over 2 ranks is even; -2 -> 1 pair: rank 1 idle),
    and a head without confidences: one all_gather_into_tensor rebuilds inference()'s result on every rank."""
    from dust3r_b200.inference import inference
    from dust3r_b200.distributed import shard_bounds
    pairs = _pairs(n_imgs)
    ref = inference(pairs, _FakeModel() if conf else _FakeModelNoConf(), 'cpu', batch_size=2, verbose=False)
    world = 2
    assert [shard_bounds(7, 3, r) for r in range(3)] == [(0, 3), (3, 5), (5, 7)]
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, world, port, n_imgs, q, conf)) for r in range(world)]
    for p in procs:
        p.start()
    got = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    conf_flag = conf
    for rank, idx1, idx2, pts, conf in got:
        assert idx1 == ref['view1']['idx'] and idx2 == ref['view2']['idx']       # bit-exact pair order
        assert np.array_equal(pts, ref['pred1']['pts3d'].numpy())
        assert np.array_equal(conf, (ref['pred2']['conf'] if conf_flag else ref['pred2']['pts3d_in_other_view']).numpy())
