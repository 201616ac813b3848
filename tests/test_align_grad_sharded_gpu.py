"""The differentiable objective on sharded scenes, on the GPU: AlignEngine.sharded_loss_and_grad (gradient pixel pass ->
all-reduce of the fixed-point accumulator block -> gradient small step -> one log-depth-gradient broadcast per owner) against
the single launch of d3r_align_loss_grad, and scene() + loss.backward() on scenes of global_aligner_sharded -- over
inference_sharded(keep='all') and keep='owned' outputs -- run by two ranks (two processes on one GPU over gloo, and two GPUs
over NCCL when the box has them) against the single-GPU scene.

Tolerances against one GPU: loss rtol 1e-5 and small-parameter gradients <= 1e-4 * max |g| per parameter kind, as in
tests/test_align_grad_gpu.py (each warp's fp32 partial sums cover other items once the item table is split, and the
fixed-point totals differ by that).  Log-depth gradients are compared bit for bit: a pixel's gradient is formed inside one
warp from its image's entries in entry order, from the same transforms, on every rank that owns the image."""
import datetime
import os
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_align_sharded_gpu import SCENES, _engine_pair, one_rank_group  # noqa: F401  (fixture)
from test_owned_rows_cpu import owned_output

pytestmark = pytest.mark.gpu

KINDS = ('im_depthmaps', 'im_poses', 'im_focals', 'im_pp', 'pw_poses', 'pw_adaptors')


# ------------------------------------------------------------------------------------- one rank: split == fused, bit for bit
@pytest.mark.parametrize('name,dist_', [('n8', 'l1'), ('n8', 'l2'), ('mixed', 'l1'), ('mixed', 'l2'), ('config5', 'l1'),
                                        ('config5', 'l2')])
@pytest.mark.parametrize('tied', [True, False])
def test_sharded_loss_and_grad_equals_fused_bit_for_bit(cuda_device, one_rank_group, name, dist_, tied):
    """Stacked and per-edge objectives, l1 / l2, tied focals and fx_and_fy; the config-5 graph (E = 1225 > 256) runs the
    multi-pass gradient step in the standalone launch.  Nothing of the optimiser state moves, and a run afterwards is the
    fused engine's."""
    if not tied and SCENES[name][1] == 'PointCloudOptimizer':
        pytest.skip('PointCloudOptimizer has one focal per image')
    make, mode, kw = SCENES[name]
    kw = dict(kw, fx_and_fy=not tied) if mode == 'ModularPointCloudOptimizer' else kw
    from dust3r_b200.cloud_opt import GlobalAlignerMode, global_aligner
    torch.manual_seed(1)
    scene = global_aligner(make(), cuda_device, mode=GlobalAlignerMode[mode], verbose=False, dist=dist_, **kw)
    fused, split = _engine_pair(scene)
    split.reset_adam()
    state = {k: getattr(split, k).clone() for k in ('logd', 'logd_m', 'logd_v', 'small', 'small_m', 'small_v')}
    got_f = fused.loss_and_grad(entry_loss=True)
    got_s = split.sharded_loss_and_grad(entry_loss=True)
    assert torch.isfinite(got_f[0]) and torch.isfinite(got_f[2]).all()
    for what, a, b in zip(('loss', 'logd_grad', 'small_grad', 'entry_loss'), got_f, got_s):
        assert torch.equal(a, b), what
    assert torch.equal(split.sharded_loss_and_grad()[0], got_f[0])          # the accumulators were left cleared
    for k, v in state.items():
        assert torch.equal(getattr(split, k), v), k
    lf, ls = fused.run(3).clone(), split.run(3).clone()
    assert torch.equal(lf, ls)
    fused.check_overflow()
    split.check_overflow()


def test_grad_entry_points_refuse_and_skip(cuda_device, one_rank_group):
    """d3r_align_grad_pixel_pass launches nothing without work items and refuses the general kernel; both halves refuse a
    null gradient buffer."""
    import ctypes as C
    from dust3r_b200 import _lib
    from dust3r_b200.cloud_opt import GlobalAlignerMode, global_aligner
    torch.manual_seed(1)
    scene = global_aligner(SCENES['n8'][0](), cuda_device, mode=GlobalAlignerMode.PointCloudOptimizer, verbose=False)
    _, split = _engine_pair(scene)
    split.prepare()
    d = split._desc()
    g = torch.full_like(split.logd, 5.0)
    d.n_items = 0
    _lib.launch(cuda_device, 'd3r_align_grad_pixel_pass', C.byref(d), g.data_ptr())
    torch.cuda.synchronize()
    assert (g == 5.0).all()
    d = split._desc()
    with pytest.raises(_lib.D3RError, match='null gradient buffer'):
        _lib.launch(cuda_device, 'd3r_align_grad_pixel_pass', C.byref(d), None)
    with pytest.raises(_lib.D3RError, match='null gradient buffer'):
        _lib.launch(cuda_device, 'd3r_align_grad_small_step', C.byref(d), None, None)
    d.stream_kernel = 0
    with pytest.raises(_lib.D3RError, match='streaming kernel only'):
        _lib.launch(cuda_device, 'd3r_align_grad_pixel_pass', C.byref(d), g.data_ptr())


# ------------------------------------------------------------------------------------- two ranks
# name -> optimizer keywords on top of SCENES': trainable adaptors and principal points; the Modular scene also has fx_and_fy,
# a preset camera and a preset focal
CASES = {'n8': dict(allow_pw_adaptors=True, optimize_pp=True),
         'mixed': dict(allow_pw_adaptors=True, optimize_pp=True),
         'config5': {}}
NITER_ADAM = 20


def _build(name, dev, sharded, seed, kind='all', nan_image=None):
    from dust3r_b200.cloud_opt import GlobalAlignerMode, global_aligner
    from dust3r_b200.distributed import global_aligner_sharded
    make, mode, kw = SCENES[name]
    out = make()
    if nan_image is not None:
        e = out['view1']['idx'].index(nan_image)
        out['pred1']['pts3d'][e][0, 0, 0] = float('nan')
    if kind == 'owned':
        out = owned_output(out, dev)
    torch.manual_seed(seed)
    build = global_aligner_sharded if sharded else global_aligner
    scene = build(out, dev, mode=GlobalAlignerMode[mode], verbose=False, **kw, **CASES[name])
    if name == 'mixed':
        scene.preset_pose([torch.eye(4)], [0])
        scene.preset_focal([30.0], [2])
    return scene


def _grads(scene):
    return {k: (None if p.grad is None else p.grad.detach().cpu().numpy().copy()) for k, p in scene.named_parameters()
            if k.split('.')[0] in KINDS}


def _params(scene):
    return {k: p.detach().cpu().numpy().copy() for k, p in scene.named_parameters() if k.split('.')[0] in KINDS}


def _backward(scene):
    scene.zero_grad(set_to_none=True)
    loss = scene()
    loss.backward()
    return float(loss.detach()), _grads(scene)


def _adam_loop(scene):
    """NITER_ADAM iterations of the reference loop body (base_opt.py:352-366) with torch.optim.Adam on scene() + backward();
    returns the losses and the parameters it ends with."""
    from dust3r_b200.cloud_opt.commons import cosine_schedule
    opt = torch.optim.Adam([p for p in scene.parameters() if p.requires_grad], lr=0.01, betas=(0.9, 0.9))
    losses = []
    for it in range(NITER_ADAM):
        for g in opt.param_groups:
            g['lr'] = cosine_schedule(it / NITER_ADAM, 0.01, 1e-6)
        opt.zero_grad()
        loss = scene()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    return np.asarray(losses), _params(scene)


def _run_case(name, kind, dev, rank, sharded):
    """Everything one rank (or the single-GPU reference) reports for one scene."""
    r = {}
    scene = _build(name, dev, sharded, seed=7 + rank, kind=kind)     # each rank draws its own start: rank 0's is evaluated
    r['owned'] = scene._get_engine().owned
    r['runs'] = [_backward(scene) for _ in range(2)]
    if SCENES[name][1] == 'ModularPointCloudOptimizer':
        with torch.no_grad():
            loss, details = scene(ret_details=True)
        r['details'] = (float(loss), details.numpy().copy())
    del scene
    nan = _build('n8', dev, sharded, seed=7, kind=kind, nan_image=7) if name == 'n8' else None
    if nan is not None:
        r['nan'] = _backward(nan) + (nan._get_engine().owned,)
        del nan
    if name != 'config5':
        scene = _build(name, dev, sharded, seed=7, kind=kind)      # every rank starts the loop from the same parameters
        losses, params = _adam_loop(scene)
        scene.compute_global_alignment(init=None, niter=10)
        fresh = _build(name, dev, sharded, seed=7, kind=kind)      # the same parameters in a scene that never ran backward()
        with torch.no_grad():
            for (k, p), (k2, q) in zip(fresh.named_parameters(), scene.named_parameters()):
                assert k == k2
                if k.split('.')[0] in KINDS:
                    p.copy_(torch.from_numpy(params[k]).to(p.device))
        fresh.compute_global_alignment(init=None, niter=10)
        r['adam'] = dict(losses=losses, params=params, cga=scene.last_losses.cpu().numpy(), cga_fresh=fresh.last_losses.cpu().numpy(),
                         final=_params(scene))
    return r


def _worker(rank, world, port, backend, names, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=600))
    try:
        dev = torch.device('cuda', rank if backend == 'nccl' else 0)
        torch.cuda.set_device(dev)
        res = {(name, kind): _run_case(name, kind, dev, rank, sharded=True) for name in names for kind in ('all', 'owned')}
        q.put((rank, res))      # numpy only
        dist.barrier()
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def _run_ranks(backend, names):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 41000 + (os.getpid() % 1500) + (0 if backend == 'gloo' else 3)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, backend, names, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(2):
        rank, res = q.get(timeout=900)
        assert not isinstance(res, str), f'rank {rank} failed:\n{res}'
        got[rank] = res
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    return [got[r] for r in range(2)]


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(a, b, equal_nan=True) if isinstance(a, np.ndarray) else a == b


def _check_grads(got, ref, what):
    assert got.keys() == ref.keys(), what
    for kind in KINDS:
        names = [k for k in ref if k.split('.')[0] == kind and ref[k] is not None]
        assert all(got[k] is None for k in ref if ref[k] is None), (what, kind)
        if not names:
            continue
        if kind == 'im_depthmaps':
            for k in names:
                assert np.array_equal(got[k], ref[k]), (what, k)
            continue
        scale = max(float(np.abs(ref[k]).max()) for k in names)
        for k in names:
            assert float(np.abs(got[k] - ref[k]).max()) <= 1e-4 * scale, (what, k)


def _check(ranks, names, device):
    for name in names:
        ref = _run_case(name, 'all', device, 0, sharded=False)
        for kind in ('all', 'owned'):
            r0, r1 = ranks[0][(name, kind)], ranks[1][(name, kind)]
            assert r0['owned'] != r1['owned']
            for r in (r0, r1):      # bit-identical across the ranks and across repeated calls
                assert all(_same(run, r0['runs'][0]) for run in r['runs']), (name, kind)
                assert _same(r.get('details'), r0.get('details')) and _same(r.get('adam'), r0.get('adam')), (name, kind)
            loss, grads = r0['runs'][0]
            ref_loss, ref_grads = ref['runs'][0]
            assert np.isfinite(loss) and abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (name, kind, loss, ref_loss)
            _check_grads(grads, ref_grads, (name, kind))
            if 'details' in ref:
                assert np.allclose(r0['details'][1], ref['details'][1], rtol=1e-5, atol=0), (name, kind)
            if 'nan' in ref:       # a NaN observation in an image of rank 1: NaN loss and small-parameter gradients everywhere
                lo, hi = r1['nan'][2]
                assert lo <= 7 < hi
                for r in (r0, r1):
                    nl, ng, _ = r['nan']
                    assert np.isnan(nl)
                    for k, g in ng.items():
                        if k.split('.')[0] != 'im_depthmaps' and g is not None:
                            assert np.isnan(g).all(), (name, kind, k)
            if 'adam' in ref:      # the custom loop: close to one GPU's; compute_global_alignment afterwards unaffected
                a, b = r0['adam'], ref['adam']
                assert np.allclose(a['losses'], b['losses'], rtol=1e-5), (name, kind)
                for k, v in b['params'].items():
                    assert float(np.abs(a['params'][k] - v).max()) < 2e-5 * NITER_ADAM, (name, kind, k)
                assert np.isfinite(a['cga']).all() and np.array_equal(a['cga'], a['cga_fresh']), (name, kind)


def test_two_ranks_on_one_gpu_gloo(cuda_device):
    names = ['n8', 'mixed']
    _check(_run_ranks('gloo', names), names, cuda_device)


def test_two_gpus_nccl(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    names = ['n8', 'mixed', 'config5']
    _check(_run_ranks('nccl', names), names, cuda_device)
