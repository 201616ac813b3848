"""Scenes aligned from the rows of inference_sharded(keep='owned') on the GPU, against global_aligner_sharded over the
all-gathered output: two processes on one GPU over gloo (and two GPUs over NCCL when the box has them), plus four processes
on one GPU for the device-memory bound.  The kept rows are routed by distributed.PairOutputRoute from each rank's slice of a
synthetic inference() result (tests/test_owned_rows_cpu.owned_output), so scenes of mixed image sizes are covered too."""
import datetime
import os
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_align_sharded_gpu import SCENES, _complete, _no_grad_loss, _params
from test_owned_rows_cpu import owned_output

pytestmark = pytest.mark.gpu

INITS = (('PointCloudOptimizer', 'mst'), ('ModularPointCloudOptimizer', 'mst'), ('ModularPointCloudOptimizer', 'known_poses'))
MEM_MARGIN = 32 << 20       # log-depths and their Adam moments, small parameters, work items, workspace, allocator rounding


def _consistent():
    from dust3r_b200.utils.synth import synth_consistent_scene
    edges = [(i, j) for i in range(6) for j in range(6) if i != j]
    out, cams, f = synth_consistent_scene(6, edges, 48, 64, seed=4)
    return out, cams, f


def _build(out, dev, mode, kw, seed):
    from dust3r_b200.cloud_opt import GlobalAlignerMode
    from dust3r_b200.distributed import global_aligner_sharded
    torch.manual_seed(seed)
    return global_aligner_sharded(out, dev, mode=GlobalAlignerMode[mode], verbose=False, **kw)


def _state(scene):
    return dict(params=_params(scene), pts3d=[p.detach().cpu().numpy() for p in scene.get_pts3d()],
                poses=scene.get_im_poses().detach().cpu().numpy(), focals=scene.get_focals().detach().cpu().numpy())


def _scenes(rank, dev):
    from dust3r_b200 import _lib
    from dust3r_b200.cloud_opt import init_im_poses
    from dust3r_b200.cloud_opt.base_opt import global_alignment_loop
    res = {}
    for name in ('n8', 'mixed', 'config5'):
        make, mode, kw = SCENES[name]
        full = make()
        for kind in ('all', 'owned'):
            out = full if kind == 'all' else owned_output(full, dev)
            scene = _build(out, dev, mode, kw, seed=7 + rank)        # each rank draws its own start: rank 0's wins
            scene.compute_global_alignment(init=None, niter=10)
            r = _state(scene)
            r.update(losses=scene.last_losses.cpu().numpy(), loss_now=_no_grad_loss(scene), owned=scene._get_engine().owned,
                     masks=[m.cpu().numpy() for m in scene.get_masks()], im_conf=[c.detach().cpu().numpy() for c in scene.im_conf])
            scene.clean_pointcloud()
            r['cleaned'] = [c.detach().cpu().numpy() for c in scene.im_conf]
            res[(name, kind)] = r
            del scene, out
    # initialisers: the spanning tree, the initial parameters and 10 iterations from them
    trees = []
    real_mst = init_im_poses.minimum_spanning_tree

    def mst(*a, **kw):
        got = real_mst(*a, **kw)
        trees.append(got[1])
        return got
    init_im_poses.minimum_spanning_tree = mst
    full, cams, f = _consistent()       # white-noise pointmaps leave PnP degenerate: the initialisers get a real scene
    for mode, init in INITS:
        for kind in ('all', 'owned'):
            out = full if kind == 'all' else owned_output(full, dev)
            scene = _build(out, dev, mode, {}, seed=7 + rank)
            if init == 'mst':
                init_im_poses.init_minimum_spanning_tree(scene)
            else:
                scene.preset_pose(cams)
                scene.preset_focal([f] * scene.n_imgs)
                init_im_poses.init_from_known_poses(scene, min_conf_thr=scene.min_conf_thr)
            r = dict(init=_params(scene), tree=trees[-1] if init == 'mst' else None)
            global_alignment_loop(scene, niter=10)
            r['losses'] = scene.last_losses.cpu().numpy()
            res[(mode, init, kind)] = r
            del scene, out
    init_im_poses.minimum_spanning_tree = real_mst
    # a NaN observation in an image of the last rank
    full = SCENES['n8'][0]()
    full['pred1']['pts3d'][full['view1']['idx'].index(7)][0, 0, 0] = float('nan')
    scene = _build(owned_output(full, dev), dev, 'PointCloudOptimizer', {}, seed=7)
    raised = False
    try:
        scene.compute_global_alignment(init=None, niter=4)
    except _lib.D3RError:
        raised = True
    res['nan'] = dict(losses=scene.last_losses.cpu().numpy(), raised=raised, owned=scene._get_engine().owned)
    return res


def _memory(rank, dev):
    """Peak device memory of alignment from kept rows, and from the full output, each from a clean start."""
    from dust3r_b200.utils.synth import synth_pair_predictions
    mode, kw = 'ModularPointCloudOptimizer', {}
    full = synth_pair_predictions(50, _complete(50), 64, 96, seed=2)
    res = {}
    for kind in ('owned', 'all'):
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        if kind == 'owned':
            out = owned_output(full, dev)
        else:           # what inference_sharded(keep='all', gather_device=cuda) leaves on every rank
            out = dict(full, pred1={k: v.to(dev) for k, v in full['pred1'].items()},
                       pred2={k: v.to(dev) for k, v in full['pred2'].items()})
        scene = _build(out, dev, mode, kw, seed=7)
        scene.compute_global_alignment(init=None, niter=10)
        torch.cuda.synchronize(dev)
        eng = scene._get_engine()
        res[kind] = dict(peak=torch.cuda.max_memory_allocated(dev) - base, obs=eng.obs.numel() * 4,
                         allocated=out['owned'].allocated if kind == 'owned' else None,
                         kept=sum(t.numel() * 4 for p in ('pred1', 'pred2') for v in out[p].values() for t in v if t is not None)
                         if kind == 'owned' else None,
                         loss=float(scene.last_losses[-1]))
        del scene, out, eng
    return res


def _worker(rank, world, port, backend, what, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=600))
    try:
        dev = torch.device('cuda', rank if backend == 'nccl' else 0)
        torch.cuda.set_device(dev)
        res = _scenes(rank, dev) if what == 'scenes' else _memory(rank, dev)
        q.put((rank, res))      # numpy only
        dist.barrier()
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def _run_ranks(backend, world, what):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 36000 + (os.getpid() % 1500) + (0 if backend == 'gloo' else 3) + 5 * world
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, what, q)) for r in range(world)]
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


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(a, b, equal_nan=True) if isinstance(a, np.ndarray) else a == b


def _check(ranks):
    for name in ('n8', 'mixed', 'config5'):
        ref = ranks[0][(name, 'all')]
        assert np.isfinite(ref['losses']).all()
        for got in ranks:
            for kind in ('all', 'owned'):      # bit-identical to the all-gathered scene, on every rank
                r = got[(name, kind)]
                for k in ('losses', 'params', 'pts3d', 'poses', 'focals', 'masks', 'im_conf', 'cleaned', 'loss_now'):
                    assert _same(r[k], ref[k]), (name, kind, k)
            assert got[(name, 'owned')]['owned'] == got[(name, 'all')]['owned']
    for name, init in INITS:
        ref = ranks[0][(name, init, 'all')]
        for got in ranks:
            a, b = got[(name, init, 'all')], got[(name, init, 'owned')]
            assert a['tree'] == b['tree'] == ref['tree']
            for k, v in a['init'].items():
                assert np.all(np.abs(b['init'][k] - v) <= 1e-6 * np.abs(v)), (name, init, k)
            assert np.isfinite(b['losses']).all() and np.allclose(b['losses'], ref['losses'], rtol=1e-5), (name, init)
    for got in ranks:
        nan = got['nan']
        assert np.isnan(nan['losses']).all() and nan['raised']
    last = ranks[-1]['nan']['owned']
    assert last[0] <= 7 < last[1]


def test_two_ranks_on_one_gpu_gloo(cuda_device):
    _check(_run_ranks('gloo', 2, 'scenes'))


def test_two_gpus_nccl(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    _check(_run_ranks('nccl', 2, 'scenes'))


def test_device_memory_bound(cuda_device):
    """Four ranks on one GPU over gloo (the reordered copy then lives in host memory): each process's peak device memory
    stays within the rows it keeps + its observations + its slice of the forward output + MEM_MARGIN; aligning from the
    all-gathered output on the same ranks exceeds that bound."""
    from dust3r_b200.distributed import shard_bounds
    world = 4
    ranks = _run_ranks('gloo', world, 'memory')
    E, row = 1225, 8 * 64 * 96 * 4
    for rank, got in enumerate(ranks):
        o, a = got['owned'], got['all']
        lo, hi = shard_bounds(E, world, rank)
        assert [name for name, dev, _ in o['allocated']] == ['send', 'recv', 'kept'] and o['allocated'][2][1] == 'cuda'
        assert o['allocated'][2][2] == o['kept']
        bound = o['kept'] + o['obs'] + (hi - lo) * row + MEM_MARGIN
        assert o['peak'] <= bound, (rank, o['peak'], bound)
        assert a['peak'] > bound, (rank, a['peak'], bound)
        assert o['loss'] == ranks[0]['owned']['loss'] == a['loss']
