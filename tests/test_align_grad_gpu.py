"""Gradients of the differentiable objective (net() + loss.backward(), d3r_align_loss_grad) against the CPU oracle's
autograd (oracle.align_oracle.loss_fn(...).backward()), tensor by tensor.  Tolerance: max |diff| <= 1e-4 * max |g_oracle| per
tensor (fp32, different summation order; the streaming kernel unprojects with MUFU exp).  Observed on an H100: small
parameters <= 3e-5, per-pixel log-depth gradients up to 3.8e-5 (config-5 graph, streaming kernel), 4e-6 .. 8e-6 on the
4-view scenes with l1."""
import copy

import numpy as np
import pytest
import torch

from dust3r_b200.utils.synth import synth_pair_predictions
from oracle.align_oracle import AlignProblem, init_params, loss_fn, pw_transforms, unproject, _dist

pytestmark = pytest.mark.gpu

KERNELS = ['stream', 'general']
SMALL = ('im_poses', 'im_focals', 'im_pp', 'pw_poses', 'pw_adaptors')


def _edges(n, symmetrize=True):
    e = [(i, j) for i in range(n) for j in range(i)]
    return e + [(j, i) for i, j in e] if symmetrize else e


def _ragged_out(shapes, edges, seed=3):
    g = torch.Generator().manual_seed(seed)
    p1 = [torch.randn(shapes[i] + (3,), generator=g) + torch.tensor([0, 0, 3.]) for i, j in edges]
    p2 = [torch.randn(shapes[j] + (3,), generator=g) + torch.tensor([0, 0, 3.]) for i, j in edges]
    c1 = [1 + 5 * torch.rand(shapes[i], generator=g) for i, j in edges]
    c2 = [1 + 5 * torch.rand(shapes[j], generator=g) for i, j in edges]
    return dict(view1=dict(idx=[i for i, j in edges]), view2=dict(idx=[j for i, j in edges]),
                pred1=dict(pts3d=p1, conf=c1), pred2=dict(pts3d_in_other_view=p2, conf=c2))


def _make(mode_name, out, P0, device, **kw):
    from dust3r_b200.cloud_opt import global_aligner, GlobalAlignerMode
    net = global_aligner(copy.deepcopy(out), device, mode=GlobalAlignerMode[mode_name], verbose=False, **kw)
    with torch.no_grad():
        if mode_name == 'PointCloudOptimizer':
            for i in range(net.n_imgs):
                net.im_depthmaps.data[i, :P0['im_depthmaps'][i].numel()] = P0['im_depthmaps'][i].to(device)
            net.im_poses.data[:] = P0['im_poses'].to(device)
            net.im_focals.data[:] = P0['im_focals'].to(device)
            net.im_pp.data[:] = P0['im_pp'].to(device)
        else:
            for i, (H, W) in enumerate(net.imshapes):
                net.im_depthmaps[i].data[:] = P0['im_depthmaps'][i].view(H, W).to(device)
                net.im_poses[i].data[:] = P0['im_poses'][i].to(device)
                net.im_focals[i].data[:] = P0['im_focals'][i].to(device)
                net.im_pp[i].data[:] = P0['im_pp'][i].to(device)
        net.pw_poses.data[:] = P0['pw_poses'].to(device)
        net.pw_adaptors.data[:] = P0['pw_adaptors'].to(device)
    return net


def _oracle(prob, P0):
    """(loss, gradients) of the reference objective by autograd, every parameter trainable."""
    P = {k: ([t.clone().requires_grad_(True) for t in v] if isinstance(v, list) else v.clone().requires_grad_(True))
         for k, v in P0.items()}
    loss = loss_fn(prob, P)
    loss.backward()
    return float(loss), {k: ([t.grad for t in v] if isinstance(v, list) else v.grad) for k, v in P.items()}


def _grads(net, mode_name):
    """.grad of the net's parameters in the oracle's layout (None where the parameter does not require grad)."""
    def stack(plist):
        g = [p.grad for p in plist]
        return None if any(x is None for x in g) else torch.stack(g).cpu()
    if mode_name == 'PointCloudOptimizer':
        g = net.im_depthmaps.grad
        depth = None if g is None else [g[i, :h * w].cpu() for i, (h, w) in enumerate(net.imshapes)]
        out = dict(im_poses=net.im_poses.grad, im_focals=net.im_focals.grad, im_pp=net.im_pp.grad)
        out = {k: (None if v is None else v.cpu()) for k, v in out.items()}
    else:
        depth = [p.grad.reshape(-1).cpu() for p in net.im_depthmaps]
        out = dict(im_poses=stack(net.im_poses), im_focals=stack(net.im_focals), im_pp=stack(net.im_pp))
    out['im_depthmaps'] = depth
    out['pw_poses'] = None if net.pw_poses.grad is None else net.pw_poses.grad.cpu()
    out['pw_adaptors'] = None if net.pw_adaptors.grad is None else net.pw_adaptors.grad.cpu()
    return out


def _margins(got, ref):
    """Observed max |diff| / max |g_oracle| per tensor (depth over all images together)."""
    m = {}
    for k in SMALL:
        if got[k] is not None:
            m[k] = float((got[k] - ref[k]).abs().max()) / max(float(ref[k].abs().max()), 1e-30)
    d = torch.cat([a - b for a, b in zip(got['im_depthmaps'], ref['im_depthmaps'])])
    m['im_depthmaps'] = float(d.abs().max()) / max(float(torch.cat(ref['im_depthmaps']).abs().max()), 1e-30)
    return m


def _check(got, ref, small_tol=1e-4, depth_tol=1e-4):
    m = _margins(got, ref)
    for k, v in m.items():
        assert v <= (depth_tol if k == 'im_depthmaps' else small_tol), (k, m)
    return m


def _backward(net):
    net.zero_grad(set_to_none=True)
    loss = net()
    assert loss.requires_grad and loss.is_cuda and loss.dim() == 0
    loss.backward()
    return float(loss.detach())


@pytest.mark.parametrize('kernel', KERNELS)
@pytest.mark.parametrize('mode_name,variant', [('PointCloudOptimizer', 'stacked'), ('ModularPointCloudOptimizer', 'per_edge')])
@pytest.mark.parametrize('dist', ['l1', 'l2'])
def test_gradients_match_oracle(cuda_device, mode_name, variant, dist, kernel):
    """Adaptors and principal points trainable; the adaptors start away from zero so their gradient is not degenerate."""
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=1)
    prob = AlignProblem.from_output(out, dist=dist, variant=variant)
    P0 = init_params(prob, seed=5)
    P0['pw_adaptors'] = 0.5 * torch.randn(P0['pw_adaptors'].shape, generator=torch.Generator().manual_seed(1))
    P0['im_pp'] = 0.3 * torch.randn(P0['im_pp'].shape, generator=torch.Generator().manual_seed(2))
    l_ref, g_ref = _oracle(prob, P0)
    net = _make(mode_name, out, P0, cuda_device, dist=dist, kernel=kernel, allow_pw_adaptors=True, optimize_pp=True)
    loss = _backward(net)
    assert net._get_engine().kernel == kernel
    assert abs(loss - l_ref) <= 1e-5 * abs(l_ref)
    print('margins', mode_name, dist, kernel, _check(_grads(net, mode_name), g_ref))


@pytest.mark.parametrize('conf', ['sqrt', 'm1', 'id'])
@pytest.mark.parametrize('kernel', KERNELS)
def test_gradients_confidence_transforms(cuda_device, conf, kernel):
    n, H, W = 3, 16, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=12)
    prob = AlignProblem.from_output(out, conf=conf)
    P0 = init_params(prob, seed=7)
    _, g_ref = _oracle(prob, P0)
    net = _make('PointCloudOptimizer', out, P0, cuda_device, conf=conf, kernel=kernel)
    _backward(net)
    _check(_grads(net, 'PointCloudOptimizer'), g_ref)


@pytest.mark.parametrize('shapes,expect', [([(24, 32), (32, 24), (16, 48)], 'stream'), ([(24, 32), (20, 36), (14, 44)], 'stream'),
                                           ([(5, 7), (9, 3), (6, 6)], 'general')])
@pytest.mark.parametrize('mode_name,variant', [('PointCloudOptimizer', 'stacked'), ('ModularPointCloudOptimizer', 'per_edge')])
def test_gradients_ragged_sizes(cuda_device, shapes, expect, mode_name, variant):
    """Different image sizes (padding of the stacked depth, partial slots, odd shapes on the general kernel), unsymmetrised
    graph, trainable adaptors and principal points.  The stacked depth's padding pixels get a zero gradient."""
    edges = [(1, 0), (2, 0), (2, 1), (0, 2)]
    out = _ragged_out(shapes, edges)
    prob = AlignProblem.from_output(out, variant=variant)
    P0 = init_params(prob, seed=9)
    _, g_ref = _oracle(prob, P0)
    net = _make(mode_name, out, P0, cuda_device, allow_pw_adaptors=True, optimize_pp=True)
    _backward(net)
    assert net._get_engine().kernel == expect
    _check(_grads(net, mode_name), g_ref)
    if mode_name == 'PointCloudOptimizer':
        g = net.im_depthmaps.grad
        for i, (h, w) in enumerate(net.imshapes):
            assert not g[i, h * w:].any()


@pytest.mark.parametrize('kernel', KERNELS)
def test_gradients_fx_and_fy(cuda_device, kernel):
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=11)
    prob = AlignProblem.from_output(out, variant='per_edge')
    P0 = init_params(prob, seed=6, fx_and_fy=True)
    P0['im_focals'] = P0['im_focals'] + torch.tensor([[0.3, -0.2]])
    _, g_ref = _oracle(prob, P0)
    net = _make('ModularPointCloudOptimizer', out, P0, cuda_device, fx_and_fy=True, kernel=kernel)
    _backward(net)
    got = _grads(net, 'ModularPointCloudOptimizer')
    assert got['im_focals'].shape == (n, 2)
    _check(got, g_ref)


@pytest.mark.parametrize('kernel', KERNELS)
def test_gradients_presets_on_a_subset(cuda_device, kernel):
    """preset_pose on two Modular images (norm_pw_scale switches off) and preset_focal on a third: their .grad stays None,
    every other gradient matches the oracle."""
    n, H, W = 4, 16, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=4)
    net0 = _make('ModularPointCloudOptimizer', out, init_params(AlignProblem.from_output(out, variant='per_edge'), seed=2),
                 cuda_device, kernel=kernel)
    poses = [torch.eye(4) for _ in range(2)]
    poses[1][:3, 3] = torch.tensor([0.3, 0.0, 0.1])
    net0.preset_pose(poses, [0, 1])
    net0.preset_focal([40.0], [2])
    assert not net0.norm_pw_scale
    prob = AlignProblem.from_output(out, variant='per_edge', norm_pw_scale=False)
    P0 = init_params(prob, seed=2)
    P0['im_poses'] = torch.stack([p.data for p in net0.im_poses]).cpu()
    P0['im_focals'] = torch.stack([p.data for p in net0.im_focals]).cpu()
    _, g_ref = _oracle(prob, P0)
    _backward(net0)
    assert net0.im_poses[0].grad is None and net0.im_poses[1].grad is None and net0.im_focals[2].grad is None
    got = _grads(net0, 'ModularPointCloudOptimizer')
    for i in (2, 3):
        assert float((net0.im_poses[i].grad.cpu() - g_ref['im_poses'][i]).abs().max()) <= 1e-4 * float(g_ref['im_poses'].abs().max())
    for i in (0, 1, 3):
        assert float((net0.im_focals[i].grad.cpu() - g_ref['im_focals'][i]).abs().max()) <= 1e-4 * float(g_ref['im_focals'].abs().max())
    got['im_poses'] = got['im_focals'] = None
    _check(got, g_ref)


@pytest.mark.parametrize('kernel', KERNELS)
def test_gradients_config5_graph(cuda_device, kernel):
    """BASELINE config 5's graph (50 views, 1225 pairs, Modular) at 64x80 pixels: the strided (multi-pass) gradient step."""
    n, H, W = 50, 64, 80
    out = synth_pair_predictions(n, _edges(n, symmetrize=False), H, W, seed=2)
    prob = AlignProblem.from_output(out, variant='per_edge')
    P0 = init_params(prob, seed=3)
    _, g_ref = _oracle(prob, P0)
    net = _make('ModularPointCloudOptimizer', out, P0, cuda_device, kernel=kernel)
    assert net.n_edges == 1225
    _backward(net)
    print('margins config5', kernel, _check(_grads(net, 'ModularPointCloudOptimizer'), g_ref))


def test_gradients_entry_window_spill(cuda_device):
    """94 entries per image, more than a streaming warp keeps in shared memory."""
    n, H, W = 48, 8, 16
    out = synth_pair_predictions(n, _edges(n, symmetrize=True), H, W, seed=8)
    prob = AlignProblem.from_output(out)
    P0 = init_params(prob, seed=4)
    _, g_ref = _oracle(prob, P0)
    net = _make('PointCloudOptimizer', out, P0, cuda_device, kernel='stream')
    eng = net._get_engine()
    assert eng.max_deg == 94 and eng.stream_window < eng.max_deg
    _backward(net)
    _check(_grads(net, 'PointCloudOptimizer'), g_ref)


def test_gradients_config3_full_size(cuda_device):
    """BASELINE config 3 at full size (8 views, 28 pairs, 512x384, PointCloudOptimizer, streaming kernel)."""
    n, H, W = 8, 384, 512
    out = synth_pair_predictions(n, _edges(n, symmetrize=False), H, W, seed=0)
    prob = AlignProblem.from_output(out)
    P0 = init_params(prob, seed=0)
    _, g_ref = _oracle(prob, P0)
    net = _make('PointCloudOptimizer', out, P0, cuda_device)
    assert net._get_engine().kernel == 'stream'
    _backward(net)
    print('margins config3', _check(_grads(net, 'PointCloudOptimizer'), g_ref))


@pytest.mark.parametrize('kernel', KERNELS)
def test_loss_bit_identical_and_state_untouched(cuda_device, kernel):
    """The gradient launch's loss equals the no_grad loss bit for bit, and a compute_global_alignment run after a backward
    is bit-identical to one without it."""
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=1)
    P0 = init_params(AlignProblem.from_output(out), seed=5)
    runs = []
    for with_grad in (False, True):
        net = _make('PointCloudOptimizer', out, P0, cuda_device, kernel=kernel)
        with torch.no_grad():
            l0 = net()
        if with_grad:
            loss = net()
            assert torch.equal(loss.detach(), l0)
            loss.backward()
        net.compute_global_alignment(init=None, niter=10)
        runs.append((net.last_losses.cpu(), [p.detach().clone() for p in net.parameters()]))
    assert torch.equal(runs[0][0], runs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


def test_autograd_semantics(cuda_device):
    """Scaled and summed losses, an extra prior term, and accumulation across backwards behave like torch."""
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=1)
    P0 = init_params(AlignProblem.from_output(out), seed=5)
    net = _make('PointCloudOptimizer', out, P0, cuda_device)
    _backward(net)
    g1 = [p.grad.clone() for p in net.parameters() if p.requires_grad]

    def grads_of(fn):
        net.zero_grad(set_to_none=True)
        fn().backward()
        return [p.grad.clone() for p in net.parameters() if p.requires_grad]
    for fn in (lambda: 3 * net(), lambda: net() + 2 * net()):
        for a, b in zip(grads_of(fn), g1):
            assert torch.allclose(a, 3 * b, rtol=1e-6, atol=0)
    lam = 1e-3
    gp = grads_of(lambda: net() + lam * net.im_focals.square().sum())
    names = [name for name, p in net.named_parameters() if p.requires_grad]
    for name, a, b in zip(names, gp, g1):
        want = b + 2 * lam * net.im_focals.detach() if name == 'im_focals' else b
        assert torch.allclose(a, want, rtol=1e-6, atol=0), name
    net.zero_grad(set_to_none=True)
    net().backward()
    net().backward()
    for p, b in zip([p for p in net.parameters() if p.requires_grad], g1):
        assert torch.equal(p.grad, 2 * b)


@pytest.mark.parametrize('mode_name', ['PointCloudOptimizer', 'ModularPointCloudOptimizer'])
def test_custom_loop_reproduces_compute_global_alignment(cuda_device, mode_name):
    """The reference loop body (base_opt.py:352-366) driven by torch.optim.Adam(betas=(0.9, 0.9)) on net() + backward():
    losses rtol 1e-5 and parameters 2e-5 * niter of the fused loop's."""
    from dust3r_b200.cloud_opt.commons import cosine_schedule
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=1)
    P0 = init_params(AlignProblem.from_output(out), seed=5)
    niter, lr0, lr_min = 10, 0.01, 1e-6
    ref = _make(mode_name, out, P0, cuda_device)
    ref.compute_global_alignment(init=None, niter=niter, lr=lr0, lr_min=lr_min)
    net = _make(mode_name, out, P0, cuda_device)
    opt = torch.optim.Adam([p for p in net.parameters() if p.requires_grad], lr=lr0, betas=(0.9, 0.9))
    losses = []
    for it in range(niter):
        for g in opt.param_groups:
            g['lr'] = cosine_schedule(it / niter, lr0, lr_min)
        opt.zero_grad()
        loss = net()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert np.allclose(losses, ref.last_losses.cpu().numpy(), rtol=1e-5), (losses, ref.last_losses)
    for (name, a), b in zip(net.named_parameters(), ref.parameters()):
        assert float((a.detach() - b.detach()).abs().max()) < 2e-5 * niter, name


def test_ret_details_matches_oracle(cuda_device):
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n, symmetrize=False), H, W, seed=3)
    prob = AlignProblem.from_output(out, variant='per_edge')
    P0 = init_params(prob, seed=1)
    net = _make('ModularPointCloudOptimizer', out, P0, cuda_device)
    loss, details = net(ret_details=True)
    assert details.device.type == 'cpu' and details.shape == (n, n)
    sR, sT, adapt = pw_transforms(prob, P0['pw_poses'], P0['pw_adaptors'])
    X = unproject(prob, P0['im_depthmaps'], P0['im_poses'], P0['im_focals'], P0['im_pp'])
    want = -torch.ones((n, n))
    for e, (i, j) in enumerate(prob.edges):
        ai = (adapt[e] * prob.pred_i[e]) @ sR[e].T + sT[e]
        aj = (adapt[e] * prob.pred_j[e]) @ sR[e].T + sT[e]
        want[i, j] = _dist(X[i], ai, prob.weight_i[e], 'l1').mean() + _dist(X[j], aj, prob.weight_j[e], 'l1').mean()
    on = want != -1
    assert torch.equal(details[~on], want[~on])
    assert torch.allclose(details[on], want[on], rtol=1e-5, atol=0)
    loss.backward()
    assert all(p.grad is not None for p in net.im_depthmaps)
