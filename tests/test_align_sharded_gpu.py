"""Sharded global alignment on the GPU: the split iteration (pixel pass -> all-reduce of the fixed-point accumulator block ->
small step, csrc/align_stream.cu) against the fused one, and scenes aligned by two ranks -- two processes on one GPU over
gloo, and two GPUs over NCCL when the box has them -- against the single-GPU run."""
import datetime
import os
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from dust3r_b200.utils.synth import synth_pair_predictions

pytestmark = pytest.mark.gpu


def _complete(n, symmetrize=False):
    e = [(i, j) for i in range(n) for j in range(i)]
    return e + [(j, i) for i, j in e] if symmetrize else e


def _mixed_output(seed=3):
    """Images of different sizes (every H*W a multiple of 4, partial last slots), unsymmetrised graph."""
    shapes = [(24, 32), (32, 24), (16, 48), (20, 36), (24, 32)]
    edges = [(1, 0), (2, 0), (2, 1), (0, 2), (3, 1), (4, 3), (4, 0), (3, 2)]
    g = torch.Generator().manual_seed(seed)
    p1 = [torch.randn(shapes[i] + (3,), generator=g) + torch.tensor([0, 0, 3.]) for i, j in edges]
    p2 = [torch.randn(shapes[j] + (3,), generator=g) + torch.tensor([0, 0, 3.]) for i, j in edges]
    c1 = [1 + 5 * torch.rand(shapes[i], generator=g) for i, j in edges]
    c2 = [1 + 5 * torch.rand(shapes[j], generator=g) for i, j in edges]
    return dict(view1=dict(idx=[i for i, j in edges]), view2=dict(idx=[j for i, j in edges]),
                pred1=dict(pts3d=p1, conf=c1), pred2=dict(pts3d_in_other_view=p2, conf=c2))


# name -> (dust3r output factory, mode, optimizer keywords)
SCENES = {
    'n8': (lambda: synth_pair_predictions(8, _complete(8), 48, 64, seed=0), 'PointCloudOptimizer', {}),
    'mixed': (_mixed_output, 'ModularPointCloudOptimizer', dict(fx_and_fy=True)),
    'config5': (lambda: synth_pair_predictions(50, _complete(50), 32, 48, seed=2), 'ModularPointCloudOptimizer', {}),
}


def _scene(name, device, sharded, seed=7, nan_image=None):
    from dust3r_b200.cloud_opt import GlobalAlignerMode, global_aligner
    from dust3r_b200.distributed import global_aligner_sharded
    make, mode, kw = SCENES[name]
    out = make()
    if nan_image is not None:          # one NaN observation in an entry of image `nan_image`
        e = out['view1']['idx'].index(nan_image)
        out['pred1']['pts3d'][e][0, 0, 0] = float('nan')
    torch.manual_seed(seed)
    build = global_aligner_sharded if sharded else global_aligner
    return build(out, device, mode=GlobalAlignerMode[mode], verbose=False, **kw)


def _params(scene):
    """Every optimised parameter of the scene as one flat numpy array per kind."""
    def flat(p):
        return torch.cat([t.detach().reshape(-1) for t in p]) if isinstance(p, torch.nn.ParameterList) else p.detach().reshape(-1)
    return {k: flat(getattr(scene, k)).cpu().numpy() for k in ('im_depthmaps', 'im_poses', 'im_focals', 'im_pp', 'pw_poses', 'pw_adaptors')}


# ------------------------------------------------------------------------------------- split == fused, one GPU
@pytest.fixture(scope='module')
def one_rank_group():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    dist.init_process_group('gloo', store=dist.HashStore(), rank=0, world_size=1)
    yield
    dist.destroy_process_group()


def _engine_pair(scene):
    """The fused engine of the scene and a sharded engine over the one-rank group, both at the scene's parameters (each
    with its own copy of the log-depths)."""
    from dust3r_b200.cloud_opt.engine import AlignEngine
    keys = scene.str_edges
    args = (scene.edges, scene.imshapes, [scene.pred_i[k] for k in keys], [scene.pred_j[k] for k in keys],
            [scene.conf_i[k] for k in keys], [scene.conf_j[k] for k in keys])
    kw = dict(device=scene.device, conf_mode=scene.conf_mode, dist=scene.dist, variant=scene._engine_variant(),
              pix_stride=scene._engine_pix_stride(), base_scale=scene.base_scale, pw_break=scene.pw_break,
              focal_break=getattr(scene, 'focal_break', getattr(scene, 'focal_brake', 20)), reverse_odd=True)
    engines = []
    for shards in (None, [(0, scene.n_imgs)]):
        eng = AlignEngine(*args, shards=shards, **kw)
        scene._engine_push(eng)
        eng.logd = eng.logd.clone()
        engines.append(eng)
    return engines


@pytest.mark.parametrize('name,dist_', [('n8', 'l1'), ('n8', 'l2'), ('mixed', 'l1'), ('mixed', 'l2'), ('config5', 'l1')])
@pytest.mark.parametrize('tied', [True, False])
def test_split_iteration_equals_fused_bit_for_bit(cuda_device, one_rank_group, name, dist_, tied):
    """Stacked (PointCloudOptimizer) and per-edge (Modular) objectives, l1 / l2, tied focals and fx_and_fy, reversed traversal
    on odd iterations; the config-5 graph (E = 1225 > 256) runs the multi-pass small step in the standalone launch."""
    if name != 'mixed' and not tied and SCENES[name][1] == 'PointCloudOptimizer':
        pytest.skip('PointCloudOptimizer has one focal per image')
    make, mode, kw = SCENES[name]
    kw = dict(kw, fx_and_fy=not tied) if mode == 'ModularPointCloudOptimizer' else kw
    from dust3r_b200.cloud_opt import GlobalAlignerMode, global_aligner
    torch.manual_seed(1)
    scene = global_aligner(make(), cuda_device, mode=GlobalAlignerMode[mode], verbose=False, dist=dist_, **kw)
    fused, split = _engine_pair(scene)
    assert split.kernel == 'stream' and split.n_items == fused.n_items and split.reduce_block[1] == 26 * scene.n_edges + 12 * scene.n_imgs + 1
    niter = 6
    lf, ls = fused.run(niter).clone(), split.run(niter).clone()
    assert torch.isfinite(lf).all() and torch.equal(lf, ls), (lf, ls)
    for attr in ('logd', 'logd_m', 'logd_v', 'small', 'small_m', 'small_v'):
        assert torch.equal(getattr(fused, attr), getattr(split, attr)), attr
    assert torch.equal(fused.evaluate_loss(), split.evaluate_loss())
    assert torch.equal(fused.pts3d(), split.pts3d())
    fused.check_overflow()
    split.check_overflow()


# ------------------------------------------------------------------------------------- two ranks
def _no_grad_loss(scene):
    with torch.no_grad():
        return float(scene())


def _worker(rank, world, port, backend, names, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        from dust3r_b200 import _lib
        dev = torch.device('cuda', rank if backend == 'nccl' else 0)
        torch.cuda.set_device(dev)
        res = {}
        for name in names:
            runs = []
            for rep in range(2):
                scene = _scene(name, dev, sharded=True, seed=7 + rank)      # each rank draws its own start: rank 0's wins
                scene.compute_global_alignment(init=None, niter=10)
                eng = scene._get_engine()
                lo, hi = eng.owned
                runs.append(dict(losses=scene.last_losses.cpu().numpy(), params=_params(scene), owned=eng.owned,
                                 n_entries=int(eng._ent_ptr[hi] - eng._ent_ptr[lo]), total_obs=eng.total_obs,
                                 pts3d=[p.detach().cpu().numpy() for p in scene.get_pts3d()],
                                 poses=scene.get_im_poses().detach().cpu().numpy(),
                                 focals=scene.get_focals().detach().cpu().numpy(), loss_now=_no_grad_loss(scene)))
            res[name] = runs
        # a NaN observation in an image of the last rank: NaN from iteration 0 on every rank, and the check raises everywhere
        scene = _scene('n8', dev, sharded=True, nan_image=7)
        raised = False
        try:
            scene.compute_global_alignment(init=None, niter=4)
        except _lib.D3RError:
            raised = True
        res['nan'] = dict(losses=scene.last_losses.cpu().numpy(), raised=raised, owned=scene._get_engine().owned)
        q.put((rank, res))      # numpy only: torch tensors would need this process alive until the parent has read them
        dist.barrier()
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def _run_ranks(backend, names):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 33000 + (os.getpid() % 1500) + (0 if backend == 'gloo' else 3)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, backend, names, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(2):
        rank, res = q.get(timeout=600)
        assert not isinstance(res, str), f'rank {rank} failed:\n{res}'
        got[rank] = res
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    return got


def _check_two_ranks(got, names, device):
    from dust3r_b200.distributed import shard_images
    for name in names:
        ref = _scene(name, device, sharded=False, seed=7)
        ref.compute_global_alignment(init=None, niter=10)
        ref_losses, ref_params = ref.last_losses.cpu().numpy(), _params(ref)
        degrees = [0] * ref.n_imgs
        for i, j in ref.edges:
            degrees[i] += 1
            degrees[j] += 1
        shards = shard_images(ref.imshapes, degrees, 2)
        a0 = got[0][name][0]
        for rank in (0, 1):
            runs = got[rank][name]
            lo, hi = runs[0]['owned']
            assert (lo, hi) == shards[rank] and hi > lo
            # this rank's observations are its own images' entries and nothing else
            assert runs[0]['n_entries'] == sum(degrees[lo:hi])
            assert runs[0]['total_obs'] == sum(degrees[i] * -(-h * w // 64) * 64 for i, (h, w) in enumerate(ref.imshapes) if lo <= i < hi)
            for run in runs:       # bit-identical across ranks and across repeated runs
                assert np.array_equal(run['losses'], a0['losses']), (name, rank)
                for k in a0['params']:
                    assert np.array_equal(run['params'][k], a0['params'][k]), (name, rank, k)
                assert all(np.array_equal(a, b) for a, b in zip(run['pts3d'], a0['pts3d']))
                assert np.array_equal(run['poses'], a0['poses']) and np.array_equal(run['focals'], a0['focals'])
                assert run['loss_now'] == a0['loss_now']
        # against the fused single-GPU run: each warp's fp32 partial covers other items once the table is split
        assert np.allclose(a0['losses'], ref_losses, rtol=1e-5), (name, a0['losses'], ref_losses)
        for k, v in ref_params.items():
            assert float(np.abs(a0['params'][k] - v).max()) < 2e-5 * 10, (name, k)
    nan = [got[r]['nan'] for r in (0, 1)]
    assert nan[1]['owned'][0] <= 7 < nan[1]['owned'][1]
    for r in nan:
        assert np.isnan(r['losses']).all() and r['raised']


def test_two_ranks_on_one_gpu_gloo(cuda_device):
    names = ['n8', 'mixed']
    got = _run_ranks('gloo', names)
    _check_two_ranks(got, names, cuda_device)


def test_two_gpus_nccl(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    names = ['n8', 'mixed', 'config5']
    got = _run_ranks('nccl', names)
    _check_two_ranks(got, names, cuda_device)
