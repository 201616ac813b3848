"""inference_sharded on a mixed-orientation scene on the GPU (8 views, 4 landscape and 4 portrait, complete symmetrised: 56
pairs of 4 size combinations), at world 1 (NCCL), with two processes on one GPU over gloo, and over NCCL on two GPUs when the
box has them.  With the small DPT model, keep='all' and keep='owned' with the results on the GPU are bit-identical to
inference() on one GPU, and 300 alignment iterations from either end where global_aligner on one GPU ends.  Random weights
give no consistent geometry for init='mst' (global_aligner on one GPU leaves the accumulator range from it), so init='mst'
runs on the consistent stand-in scene of tests/test_mixed_sharded_cpu.py, computed on the GPU, through the same path."""
import datetime
import os
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _pairs(H, W):
    from dust3r_b200.image_pairs import make_pairs
    from dust3r_b200.utils.synth import synth_images
    views = [dict(synth_images(1, *hw, seed=70 + k)[0], idx=k, instance=str(k)) for k, hw in enumerate([(H, W), (W, H)] * 4)]
    return make_pairs(views, scene_graph='complete', prefilter=None, symmetrize=True)


def _align(outs, dev, init):
    """300 iterations from `init` on one GPU (global_aligner over inference()'s result) and on the group (global_aligner_sharded
    over each keep mode's output): final loss and parameters."""
    from dust3r_b200.cloud_opt import global_aligner
    from dust3r_b200.distributed import global_aligner_sharded
    from test_align_sharded_gpu import _params
    res = {}
    for kind, out in zip(('single', 'all', 'owned'), outs):
        torch.manual_seed(7)
        scene = (global_aligner if kind == 'single' else global_aligner_sharded)(out, dev, verbose=False)
        loss = scene.compute_global_alignment(init=init, niter=300)
        res[kind] = dict(loss=float(loss), params=_params(scene))
    return res


def _check_outputs(pairs, net, dev):
    """Both keep modes with gather_device on the GPU against inference() on this rank's GPU, bit for bit; returns the three."""
    from dust3r_b200.distributed import inference_sharded, pair_graph, shard_images
    from dust3r_b200.inference import inference
    from dust3r_b200.utils.device import to_cpu
    from test_mixed_sharded_cpu import _assert_same
    ref = inference(pairs, net, dev, batch_size=4, verbose=False, keep_on_device=True)
    assert isinstance(ref['pred1']['pts3d'], list) and ref['pred1']['pts3d'][0].device == dev
    full = inference_sharded(pairs, net, dev, batch_size=4, verbose=False, gather_device=dev)
    for which in ('pred1', 'pred2'):
        _assert_same(full[which], ref[which], which)
    for v in ('view1', 'view2'):
        _assert_same(to_cpu(full[v]), to_cpu(ref[v]), v)
    owned = inference_sharded(pairs, net, dev, batch_size=4, verbose=False, gather_device=dev, keep='owned')
    edges, imshapes = pair_graph(pairs)
    degrees = np.bincount(np.asarray(edges).reshape(-1), minlength=len(imshapes)).tolist()
    lo, hi = shard_images(imshapes, degrees, dist.get_world_size())[dist.get_rank()]
    assert owned['owned'].shards[dist.get_rank()] == (lo, hi)
    for which in ('pred1', 'pred2'):
        assert sorted(owned[which]) == sorted(ref[which])
        for key, rows in owned[which].items():
            for e, (i, j) in enumerate(edges):
                if lo <= i < hi or (which == 'pred2' and lo <= j < hi):
                    _assert_same(rows[e], ref[which][key][e], f'{which}.{key}[{e}]')
                else:
                    assert rows[e] is None, (which, key, e)
    return ref, full, owned


def _worker(rank, world, port, backend, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    try:
        dev = torch.device('cuda', rank if backend == 'nccl' else 0)
        torch.cuda.set_device(dev)
        kw = dict(device_id=dev) if backend == 'nccl' else {}
        dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=600), **kw)
        from test_forward_gpu import _build, _small_cfgs
        from test_mixed_sharded_cpu import _SceneModel
        cfg, H, W = _small_cfgs()['small_dpt']
        net, _ = _build(cfg, 11, dev)
        pairs = _pairs(H, W)
        res = dict(dpt=_align(_check_outputs(pairs, net, dev), dev, init=None),
                   scene=_align(_check_outputs(pairs, _SceneModel(), dev), dev, init='mst'))
        q.put((rank, res))      # numpy only
        dist.barrier()
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _run_ranks(backend, world):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 38000 + (os.getpid() % 1500) + (0 if backend == 'gloo' else 3) + 5 * world
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        rank, res = q.get(timeout=900)
        assert not isinstance(res, str), f'rank {rank} failed:\n{res}'
        got[rank] = res
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    return [got[r] for r in range(world)]


def _check(ranks, world):
    for case in ('dpt', 'scene'):
        ref = ranks[0][case]['single']
        assert np.isfinite(ref['loss'])
        for got in ranks:
            assert got[case]['single']['loss'] == ref['loss']
            for kind in ('all', 'owned'):
                r, r0 = got[case][kind], ranks[0][case][kind]
                # the same scene on every rank, bit for bit
                assert r['loss'] == r0['loss'] and all(np.array_equal(v, r0['params'][k]) for k, v in r['params'].items())
                if world == 1 and case == 'dpt':    # a group of one runs global_aligner itself
                    assert r['loss'] == ref['loss'], (case, kind)
                    assert all(np.array_equal(v, ref['params'][k]) for k, v in r['params'].items()), (case, kind)
                else:   # the tolerances of the sharded alignment against the fused single-GPU run; init='mst' is not
                        # bit-reproducible on the GPU (its registration moments are summed with atomics)
                    assert np.isclose(r['loss'], ref['loss'], rtol=1e-5), (case, kind, r['loss'], ref['loss'])
                    for k, v in ref['params'].items():
                        assert float(np.abs(r['params'][k] - v).max()) < 2e-5 * 10, (case, kind, k)


@pytest.mark.timeout(1200)
def test_world_one_nccl(cuda_device):
    _check(_run_ranks('nccl', 1), 1)


@pytest.mark.timeout(1200)
def test_two_ranks_on_one_gpu_gloo(cuda_device):
    _check(_run_ranks('gloo', 2), 2)


@pytest.mark.timeout(1200)
def test_two_gpus_nccl(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    _check(_run_ranks('nccl', 2), 2)
