"""Parity of the fused CUDA alignment step (through the C ABI / global_aligner API) against the CPU
oracle (oracle/align_oracle.py) and the reference goldens.  fp32 path: tolerances are stated per test.
The kernel uses a different (deterministic, tree) summation order than torch autograd, and Adam's
g/sqrt(v) normalisation amplifies last-bit gradient differences of near-zero gradients, so
parameters are compared with absolute tolerances that grow with the iteration count."""
import copy
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from dust3r_b200.utils.synth import synth_pair_predictions
from oracle.align_oracle import AlignProblem, init_params, align_oracle

pytestmark = pytest.mark.gpu


def _edges(n, symmetrize=True):
    e = [(i, j) for i in range(n) for j in range(i)]
    return e + [(j, i) for i, j in e] if symmetrize else e


def _make(mode_name, out, P0, device, **kw):
    from dust3r_b200.cloud_opt import global_aligner, GlobalAlignerMode
    net = global_aligner(copy.deepcopy(out), device, mode=GlobalAlignerMode[mode_name], verbose=False, **kw)
    n = net.n_imgs
    with torch.no_grad():
        if mode_name == 'PointCloudOptimizer':
            for i in range(n):
                net.im_depthmaps.data[i, :P0['im_depthmaps'][i].numel()] = P0['im_depthmaps'][i].to(device)
            net.im_poses.data[:] = P0['im_poses'].to(device)
            net.im_focals.data[:] = P0['im_focals'].to(device)
        else:
            for i, (H, W) in enumerate(net.imshapes):
                net.im_depthmaps[i].data[:] = P0['im_depthmaps'][i].view(H, W).to(device)
                net.im_poses[i].data[:] = P0['im_poses'][i].to(device)
                net.im_focals[i].data[:] = P0['im_focals'][i].to(device)
        net.pw_poses.data[:] = P0['pw_poses'].to(device)
    return net


def _final(net, mode_name):
    if mode_name == 'PointCloudOptimizer':
        depth = [net.im_depthmaps.data[i, :h * w].cpu() for i, (h, w) in enumerate(net.imshapes)]
        return depth, net.im_poses.data.cpu(), net.im_focals.data.cpu(), net.pw_poses.data.cpu()
    depth = [d.data.reshape(-1).cpu() for d in net.im_depthmaps]
    return (depth, torch.stack([p.data for p in net.im_poses]).cpu(),
            torch.stack([p.data for p in net.im_focals]).cpu(), net.pw_poses.data.cpu())


KERNELS = ['stream', 'general']   # csrc/align_stream.cu (what real image sizes run) and csrc/align_step.cu (any shape)


@pytest.mark.parametrize('kernel', KERNELS)
@pytest.mark.parametrize('mode_name,variant', [('PointCloudOptimizer', 'stacked'), ('ModularPointCloudOptimizer', 'per_edge')])
@pytest.mark.parametrize('dist', ['l1', 'l2'])
def test_first_iterations_match_oracle(cuda_device, mode_name, variant, dist, kernel):
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=1)
    prob = AlignProblem.from_output(out, dist=dist, variant=variant)
    P0 = init_params(prob, seed=5)
    for niter in (1, 3, 10):
        losses_ref, fin = align_oracle(prob, P0, niter=niter)
        net = _make(mode_name, out, P0, cuda_device, dist=dist, kernel=kernel)
        loss = net.compute_global_alignment(init=None, niter=niter, schedule='cosine', lr=0.01)
        assert net._get_engine().kernel == kernel
        got = net.last_losses.cpu().numpy()
        assert np.allclose(got, losses_ref, rtol=1e-5), (niter, got, losses_ref)
        assert abs(loss - losses_ref[-1]) <= 1e-5 * abs(losses_ref[-1])
        depth, poses, focals, pw = _final(net, mode_name)
        tol = 2e-5 * niter + 1e-6
        assert max(float((a - b).abs().max()) for a, b in zip(depth, fin['im_depthmaps'])) < tol
        assert float((poses - fin['im_poses']).abs().max()) < tol
        assert float((focals - fin['im_focals']).abs().max()) < tol
        assert float((pw - fin['pw_poses']).abs().max()) < tol


@pytest.mark.parametrize('variant,mode_name', [('stacked', 'PointCloudOptimizer'), ('per_edge', 'ModularPointCloudOptimizer')])
@pytest.mark.parametrize('dist', ['l1', 'l2'])
@pytest.mark.parametrize('schedule', ['cosine', 'linear'])
@pytest.mark.parametrize('kernel', KERNELS)
def test_matches_reference_golden_60_iters(cuda_device, variant, mode_name, dist, schedule, kernel):
    """golden = the reference's own loop (+ local roma restatement), 60 iterations."""
    gold = np.load(os.path.join(GOLDEN, 'align_n4.npz'))
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=1)
    prob = AlignProblem.from_output(out, dist=dist, variant=variant)
    P0 = init_params(prob, seed=5)
    net = _make(mode_name, out, P0, cuda_device, dist=dist, kernel=kernel)
    net.compute_global_alignment(init=None, niter=60, schedule=schedule, lr=0.01)
    key = f'{variant}|{dist}|{schedule}'
    got = net.last_losses.cpu().numpy()
    assert np.allclose(got, gold[key + '|loss'], rtol=2e-4), float(np.abs(got / gold[key + '|loss'] - 1).max())
    depth, poses, focals, pw = _final(net, mode_name)
    assert np.abs(torch.stack(depth).numpy() - gold[key + '|depth']).max() < 5e-3
    assert np.abs(poses.numpy() - gold[key + '|poses']).max() < 5e-3
    assert np.abs(pw.numpy() - gold[key + '|pw']).max() < 5e-3
    assert np.abs(focals.numpy() - gold[key + '|focals']).max() < 5e-3


@pytest.mark.parametrize('shapes,expect', [([(24, 32), (32, 24), (16, 48)], 'stream'), ([(24, 32), (20, 36), (14, 44)], 'stream'),
                                           ([(5, 7), (9, 3), (6, 6)], 'general')])
def test_ragged_image_sizes_and_adaptors_and_pp(cuda_device, shapes, expect):
    """Different image sizes (padding path, partial last slots, odd pixel counts -> general kernel), trainable adaptors
    and principal points, unsymmetrised graph."""
    from dust3r_b200.cloud_opt import global_aligner, GlobalAlignerMode
    edges = [(1, 0), (2, 0), (2, 1), (0, 2)]
    g = torch.Generator().manual_seed(3)
    p1 = [torch.randn(shapes[i] + (3,), generator=g) + torch.tensor([0, 0, 3.]) for i, j in edges]
    p2 = [torch.randn(shapes[j] + (3,), generator=g) + torch.tensor([0, 0, 3.]) for i, j in edges]
    c1 = [1 + 5 * torch.rand(shapes[i], generator=g) for i, j in edges]
    c2 = [1 + 5 * torch.rand(shapes[j], generator=g) for i, j in edges]
    out = dict(view1=dict(idx=[i for i, j in edges]), view2=dict(idx=[j for i, j in edges]),
               pred1=dict(pts3d=p1, conf=c1), pred2=dict(pts3d_in_other_view=p2, conf=c2))
    for mode_name, variant in (('PointCloudOptimizer', 'stacked'), ('ModularPointCloudOptimizer', 'per_edge')):
        prob = AlignProblem.from_output(out, dist='l1', variant=variant)
        P0 = init_params(prob, seed=9)
        trainable = ('im_depthmaps', 'im_poses', 'im_focals', 'pw_poses', 'im_pp', 'pw_adaptors')
        losses_ref, fin = align_oracle(prob, P0, niter=5, trainable=trainable)
        net = _make(mode_name, out, P0, cuda_device, dist='l1', allow_pw_adaptors=True, optimize_pp=True)
        net.compute_global_alignment(init=None, niter=5)
        assert net._get_engine().kernel == expect
        assert np.allclose(net.last_losses.cpu().numpy(), losses_ref, rtol=1e-5)
        depth, poses, focals, pw = _final(net, mode_name)
        assert max(float((a - b).abs().max()) for a, b in zip(depth, fin['im_depthmaps'])) < 2e-4
        assert float((pw - fin['pw_poses']).abs().max()) < 2e-4
        assert float((net.pw_adaptors.data.cpu() - fin['pw_adaptors']).abs().max()) < 2e-4
        pp = net.im_pp.data.cpu() if mode_name == 'PointCloudOptimizer' else torch.stack([p.data for p in net.im_pp]).cpu()
        assert float((pp - fin['im_pp']).abs().max()) < 2e-4


def test_frozen_poses_and_focals(cuda_device):
    """preset_pose / preset_focal freeze parameters (optimizer.py:66-91): they must not move, and
    norm_pw_scale switches off."""
    n, H, W = 3, 16, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=4)
    prob = AlignProblem.from_output(out, dist='l1', variant='stacked', norm_pw_scale=False)
    P0 = init_params(prob, seed=2)
    net = _make('PointCloudOptimizer', out, P0, cuda_device)
    poses = [torch.eye(4) for _ in range(n)]
    for i in range(n):
        poses[i][:3, 3] = torch.tensor([0.1 * i, 0.0, 0.2 * i])
    net.preset_pose(poses)
    net.preset_focal([40.0] * n)
    P0['im_poses'] = net.im_poses.data.cpu().clone()
    P0['im_focals'] = net.im_focals.data.cpu().clone()
    losses_ref, fin = align_oracle(prob, P0, niter=8, trainable=('im_depthmaps', 'pw_poses'))
    net.compute_global_alignment(init=None, niter=8)
    assert np.allclose(net.last_losses.cpu().numpy(), losses_ref, rtol=1e-5)
    assert torch.equal(net.im_poses.data.cpu(), P0['im_poses']) and torch.equal(net.im_focals.data.cpu(), P0['im_focals'])
    assert float((net.pw_poses.data.cpu() - fin['pw_poses']).abs().max()) < 2e-4


def test_full_size_properties(cuda_device):
    """BASELINE config 3 size (8 views, 28 pairs, 512x384): size-independent properties —
    forward() equals the first loop loss, the loss decreases, runs are bit-reproducible (the
    reduction tree is deterministic), pointmaps are finite."""
    n, H, W = 8, 384, 512
    out = synth_pair_predictions(n, _edges(n, symmetrize=False), H, W, seed=0)
    from dust3r_b200.cloud_opt import global_aligner
    runs = []
    for rep in range(2):
        torch.manual_seed(7)
        net = global_aligner(copy.deepcopy(out), cuda_device, verbose=False)
        l0 = float(net())
        net.compute_global_alignment(init=None, niter=30)
        ls = net.last_losses.cpu().numpy()
        assert abs(l0 - ls[0]) <= 1e-6 * abs(l0)
        assert ls[-1] < ls[0] and np.isfinite(ls).all()
        assert all(torch.isfinite(p).all() for p in net.get_pts3d())
        runs.append((ls, net.im_depthmaps.data.clone(), net.pw_poses.data.clone()))
    assert np.array_equal(runs[0][0], runs[1][0])
    assert torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][2], runs[1][2])


def test_get_pts3d_matches_oracle_unprojection(cuda_device):
    from oracle.align_oracle import unproject
    n, H, W = 3, 24, 40
    out = synth_pair_predictions(n, _edges(n), H, W, seed=6)
    prob = AlignProblem.from_output(out)
    P0 = init_params(prob, seed=1)
    net = _make('PointCloudOptimizer', out, P0, cuda_device)
    ref = unproject(prob, P0['im_depthmaps'], P0['im_poses'], P0['im_focals'], P0['im_pp'])
    for a, b in zip(net.get_pts3d(), ref):
        assert torch.allclose(a.cpu().reshape(-1, 3), b, rtol=1e-5, atol=1e-6)


def test_config3_full_size_10_iterations_match_oracle(cuda_device):
    """BASELINE config 3 at full size (8 views -> 28 pairs at 512x384, PointCloudOptimizer): 10 iterations of the
    fused step against the CPU oracle loop (autograd + torch.optim.Adam).  fp32: losses rtol 1e-5, parameters
    abs 2e-5 * niter."""
    n, H, W = 8, 384, 512
    out = synth_pair_predictions(n, _edges(n, symmetrize=False), H, W, seed=0)
    prob = AlignProblem.from_output(out)
    P0 = init_params(prob, seed=0)
    niter = 10
    losses_ref, fin = align_oracle(prob, P0, niter=niter)
    for kernel in KERNELS:
        net = _make('PointCloudOptimizer', out, P0, cuda_device, kernel=kernel)
        net.compute_global_alignment(init=None, niter=niter)
        got = net.last_losses.cpu().numpy()
        assert np.allclose(got, losses_ref, rtol=1e-5), (kernel, got, losses_ref)
        depth, poses, focals, pw = _final(net, 'PointCloudOptimizer')
        tol = 2e-5 * niter
        assert max(float((a - b).abs().max()) for a, b in zip(depth, fin['im_depthmaps'])) < tol
        assert float((poses - fin['im_poses']).abs().max()) < tol and float((pw - fin['pw_poses']).abs().max()) < tol
        assert float((focals - fin['im_focals']).abs().max()) < tol


def test_config5_graph_50_views_1225_pairs_modular_matches_oracle(cuda_device):
    """BASELINE config 5's graph (50 views -> 1225 pairs, symmetrize=False, ModularPointCloudOptimizer): 3 iterations
    against the CPU oracle.  The graph, entry degrees (49 per image) and work decomposition are the benchmark's; the
    images are 128x160 so that the autograd oracle (which keeps ~15 (P,3) tensors per edge) fits the host."""
    n, H, W = 50, 128, 160
    out = synth_pair_predictions(n, _edges(n, symmetrize=False), H, W, seed=2)
    prob = AlignProblem.from_output(out, variant='per_edge')
    P0 = init_params(prob, seed=3)
    losses_ref, fin = align_oracle(prob, P0, niter=3)
    for kernel in KERNELS:
        net = _make('ModularPointCloudOptimizer', out, P0, cuda_device, kernel=kernel)
        assert net.n_edges == 1225 and net._get_engine().kernel == kernel
        net.compute_global_alignment(init=None, niter=3)
        assert np.allclose(net.last_losses.cpu().numpy(), losses_ref, rtol=1e-5), kernel
        depth, poses, focals, pw = _final(net, 'ModularPointCloudOptimizer')
        assert max(float((a - b).abs().max()) for a, b in zip(depth, fin['im_depthmaps'])) < 1e-4, kernel
        assert float((poses - fin['im_poses']).abs().max()) < 1e-4 and float((pw - fin['pw_poses']).abs().max()) < 1e-4, kernel


def test_stream_kernel_entry_window_spill(cuda_device):
    """More entries per image (94) than a warp keeps in shared memory (window 92): the partial sums of a window leave
    the SM before the next one starts."""
    n, H, W = 48, 8, 16
    out = synth_pair_predictions(n, _edges(n, symmetrize=True), H, W, seed=8)
    prob = AlignProblem.from_output(out)
    P0 = init_params(prob, seed=4)
    losses_ref, fin = align_oracle(prob, P0, niter=2)
    net = _make('PointCloudOptimizer', out, P0, cuda_device, kernel='stream')
    eng = net._get_engine()
    assert eng.max_deg == 94 and eng.stream_window < eng.max_deg
    net.compute_global_alignment(init=None, niter=2)
    assert np.allclose(net.last_losses.cpu().numpy(), losses_ref, rtol=1e-5)
    assert float((net.pw_poses.data.cpu() - fin['pw_poses']).abs().max()) < 1e-4


@pytest.mark.parametrize('kernel', KERNELS)
def test_modular_fx_and_fy(cuda_device, kernel):
    """fx_and_fy=True (modular_optimizer.py:24-33): two focal parameters per image, each with its own gradient."""
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=11)
    prob = AlignProblem.from_output(out, variant='per_edge')
    P0 = init_params(prob, seed=6, fx_and_fy=True)
    P0['im_focals'] = P0['im_focals'] + torch.tensor([[0.3, -0.2]])      # start with fx != fy
    losses_ref, fin = align_oracle(prob, P0, niter=6)
    net = _make('ModularPointCloudOptimizer', out, P0, cuda_device, fx_and_fy=True, kernel=kernel)
    assert tuple(net.im_focals[0].shape) == (2,)
    net.compute_global_alignment(init=None, niter=6)
    assert np.allclose(net.last_losses.cpu().numpy(), losses_ref, rtol=1e-5)
    focals = torch.stack([p.data for p in net.im_focals]).cpu()
    assert float((focals - fin['im_focals']).abs().max()) < 2e-4
    assert float((focals[:, 0] - focals[:, 1]).abs().min()) > 1e-3        # the two focals really evolve separately
    K = net.get_intrinsics()
    assert torch.allclose(K[:, 0, 0].cpu(), torch.exp(focals[:, 0] / 20)) and torch.allclose(K[:, 1, 1].cpu(), torch.exp(focals[:, 1] / 20))


@pytest.mark.parametrize('conf', ['sqrt', 'm1', 'id'])
def test_confidence_transforms(cuda_device, conf):
    """conf = 'log' is the default everywhere else; the other transforms of commons.py:73-80 are applied by the
    packing kernel."""
    n, H, W = 3, 16, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=12)
    prob = AlignProblem.from_output(out, conf=conf)
    P0 = init_params(prob, seed=7)
    losses_ref, _ = align_oracle(prob, P0, niter=4)
    for kernel in KERNELS:
        net = _make('PointCloudOptimizer', out, P0, cuda_device, conf=conf, kernel=kernel)
        net.compute_global_alignment(init=None, niter=4)
        assert np.allclose(net.last_losses.cpu().numpy(), losses_ref, rtol=1e-5), (conf, kernel)


def test_device_resident_predictions_are_packed_in_place(cuda_device):
    """global_aligner on predictions that already live in HBM (inference(keep_on_device=True) / all-gather output):
    nothing goes through the host, the per-edge dictionaries are views of the 4 stacked tensors, and the result is
    bit-identical to the host-input path."""
    from dust3r_b200.cloud_opt import global_aligner
    n, H, W = 4, 32, 48
    out = synth_pair_predictions(n, _edges(n), H, W, seed=13)
    dev_out = copy.deepcopy(out)
    for side, keys in (('pred1', ('pts3d', 'conf')), ('pred2', ('pts3d_in_other_view', 'conf'))):
        for k in keys:
            dev_out[side][k] = dev_out[side][k].to(cuda_device)
    losses = []
    for o in (out, dev_out):
        torch.manual_seed(5)
        net = global_aligner(copy.deepcopy(o), cuda_device, verbose=False)
        base = net._obs_stacks[0]
        assert base.is_cuda and net.pred_i[net.str_edges[1]].data_ptr() == base[1].data_ptr()
        net.compute_global_alignment(init=None, niter=5)
        losses.append(net.last_losses.cpu().numpy())
    assert np.array_equal(losses[0], losses[1])
