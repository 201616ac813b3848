"""The global-alignment kernels element by element against the float64 oracle of oracle/align_float64.py.

Every case reads back what the kernel read (packed observations, fp32 parameters, log-depths, item table), evaluates
the objective in float64, and requires |kernel - float64| <= bound for EVERY element of: dL/dlog-depth per pixel, the
(E, 2) per-entry losses, the total loss and dL/d(small parameter).  The bounds, their constants and where they come from
are written out in oracle/align_float64.py's docstring; nothing is tuned to the observations.  Every case prints its
worst err / bound per quantity and the share of the small-gradient bound that is fixed-point quantisation (2^-41 per
fix_add partial).  Padding pixels of the stacked depth must get a gradient of exactly 0.

The resolution demonstration (ragged streaming case): three kernel mistakes built on the float64 side -- one pixel
unprojected one column off at a row wrap inside a pixel pair, one entry's contribution dropped at the pixel with the
smallest nonzero gradient, one pixel missing from one entry's sums -- each exceeds the element-wise bound and each stays
inside the per-tensor `1e-4 * max |g|` criterion of tests/test_align_grad_gpu.py.  The scene has a block of
low-confidence pixels, which is where that criterion is blind.

Also here: the packing kernel against a numpy re-pack (both layouts, every confidence transform), eng.pts3d() against
float64 unprojection, and the overflow / NaN contract: a NaN observation or a scene whose partial sums leave the 2^18
fixed-point range gives a NaN loss and NaN small gradients from net() and backward(), and compute_global_alignment
raises (the log-depth gradients are not poisoned and may stay finite); an in-range scene 100x larger than usual stays
inside the bounds.

The Adam step, element by element (check_adam_step): after iterations [0, k), every log-depth, exp_avg and exp_avg_sq
and every trainable small parameter and its moments after iteration k against a float64 Adam step from the snapshot,
the exported gradient and the fp32 schedule row (oracle.align_float64.adam64 gives the bound), for k = 0, an odd k
(reversed item table) and an even k on both kernels; non-trainable entries and their moments, and the padding pixels
of the stacked depth and its moments, are bit-unchanged, and tied focals stay equal.  At k = 0 the moments are one
rounding of the gradient, so the test asserts that the gradient launch and the training iteration compute the same gd
bit for bit.

Covered at full size: config 3 (8 views, 28 pairs, 512x384, streaming kernel): per-pixel, loss and small-parameter
bounds and the Adam step at k = 1.  Config 5's graph (50 views, 1225 pairs, Modular) runs at 64x80.

Observed on one H100 80GB HBM3 (400 W power limit); no constant was fitted to these.  Gradients and losses: worst
err / bound between 1e-4 (total loss) and 0.13 (small gradients of the scene around the entry window), per-pixel
gradients 0.01 .. 0.11.  The total loss sits lowest because its bound adds every entry's worst case while the entries'
actual rounding errors, of either sign, largely cancel in the sum.  Adam step: log-depths 0.66 .. 0.75 -- dominated by
the final rounding of a value near -3, which is half an ulp (2^-23) against u |p| ~ 1.7e-7 in the bound, a fixed
ratio of exact arithmetic rather than a tuned constant; exp_avg / exp_avg_sq 0.23 .. 0.48, small parameters 0.03 .. 0.54,
their moments <= 0.02.  The fixed-point share of the small-gradient bound is largest at config-5 coefficients: max
0.9 %, median 0.25 % on the streaming kernel (0.1 % / 0.03 % on the general kernel), so quantisation is not what limits
the small gradients today.  The file runs in about 40 s there, most of it the float64 oracle on the CPU."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from dust3r_b200 import _lib
from dust3r_b200.utils.synth import synth_pair_predictions
from oracle import align_float64 as A
from oracle.align_oracle import AlignProblem, init_params

pytestmark = pytest.mark.gpu

KERNELS = ['stream', 'general']
MODES = [('PointCloudOptimizer', 'stacked'), ('ModularPointCloudOptimizer', 'per_edge')]


def _edges(n, symmetrize=True):
    e = [(i, j) for i in range(n) for j in range(i)]
    return e + [(j, i) for i, j in e] if symmetrize else e


def _ragged_out(shapes, edges, seed=3, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    p1 = [scale * (torch.randn(shapes[i] + (3,), generator=g) + torch.tensor([0, 0, 3.])) for i, j in edges]
    p2 = [scale * (torch.randn(shapes[j] + (3,), generator=g) + torch.tensor([0, 0, 3.])) for i, j in edges]
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


def _params(out, variant, seed, fx_and_fy=False, away_from_zero=True):
    P0 = init_params(AlignProblem.from_output(out, variant=variant), seed=seed, fx_and_fy=fx_and_fy)
    if away_from_zero:
        P0['pw_adaptors'] = 0.5 * torch.randn(P0['pw_adaptors'].shape, generator=torch.Generator().manual_seed(1))
        P0['im_pp'] = 0.3 * torch.randn(P0['im_pp'].shape, generator=torch.Generator().manual_seed(2))
    return P0


def _engine(net):
    eng = net._get_engine()
    net._engine_push(eng)
    return eng


def check_bounds(eng, label, demo_img=None, grads=None):
    """Runs one gradient launch and checks every element against the float64 oracle; returns the report, and with
    `grads` (a dict) fills in the exported gradients and the small-gradient bound."""
    loss, gd, sg, ent = eng.loss_and_grad(entry_loss=True)
    if grads is not None:
        grads.update(logd=gd.clone(), small=sg.clone())
    sc = A.scene_from_engine(eng)
    T = A.terms(sc)
    rep = {}
    gd = gd.double().cpu()
    worst = 0.0
    for i in range(sc.n):
        a, P = int(eng.pix_off[i]), eng.areas[i]
        got = gd[a:a + P]
        assert not gd[a + P:int(eng.pix_off[i + 1])].any(), 'padding pixels must get a zero gradient'
        r = A.ratio((got - T['gd'][i]).abs(), T['gd_bound'][i])
        worst = max(worst, r)
    rep['logd_grad'] = worst
    L, Lb, l_tot, l_tot_b = A.loss_bounds(sc, T)
    ent = ent.double().cpu()
    got_ent = torch.stack([ent[int(e), int(s)] for e, s in zip(sc.ent_edge, sc.ent_side)])
    rep['entry_loss'] = A.ratio((got_ent - L).abs(), Lb)
    rep['loss'] = abs(float(loss) - l_tot) / l_tot_b
    l64, g64 = A.small_grad64(sc)
    sb, fixed = A.small_bound(sc, T)
    err = (sg.double().cpu() - g64).abs()
    rep['small_grad'] = A.ratio(err, sb)
    worst_small = int(torch.where(err == 0, torch.zeros_like(err), err / sb).argmax())
    if grads is not None:
        grads['small_bound'] = sb
    share = fixed[sb > 0] / sb[sb > 0]
    rep['fixed_point_share_max'] = float(share.max())
    rep['fixed_point_share_median'] = float(share.median())
    o = sc.offsets()
    kind = max((v, k) for k, v in o.items() if k != 'total' and v <= worst_small)[1]
    print(f'\n[{label}] worst err/bound: ' + ', '.join(f'{k}={v:.3g}' for k, v in rep.items())
          + f' (worst small element: {kind} + {worst_small - o[kind]})')
    for k in ('logd_grad', 'entry_loss', 'loss', 'small_grad'):
        assert rep[k] <= 1.0, (label, k, rep)
    if demo_img is not None:
        demo = A.resolution_demo(sc, T, sb, g64, img=demo_img)
        print(f'[{label}] mutations (err/bound, err/(1e-4 max|g|)):', demo)
        for name, (caught, missed) in demo.items():
            assert caught > 1, (name, 'the element-wise bound must see the mutation', caught)
            assert missed <= 1, (name, 'the per-tensor criterion is expected to miss it', missed)
    return rep


@pytest.mark.parametrize('dist', ['l1', 'l2'])
@pytest.mark.parametrize('mode_name,variant', MODES)
@pytest.mark.parametrize('kernel', KERNELS)
def test_baseline_every_gradient_kind(cuda_device, kernel, mode_name, variant, dist):
    """4 views 24x32, symmetric graph, adaptors and principal points trainable and away from 0."""
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=1)
    net = _make(mode_name, out, _params(out, variant, 5), cuda_device, dist=dist, kernel=kernel,
                allow_pw_adaptors=True, optimize_pp=True)
    eng = _engine(net)
    assert eng.kernel == kernel
    check_bounds(eng, f'baseline {kernel} {variant} {dist}')


RAGGED = [(24, 32), (20, 36), (14, 44), (48, 16), (12, 100), (12, 33)]
RAGGED_EDGES = [(1, 0), (2, 0), (2, 1), (0, 2), (3, 2), (4, 3), (0, 4), (5, 4), (5, 0), (1, 5)]


@pytest.mark.parametrize('dist', ['l1', 'l2'])
@pytest.mark.parametrize('mode_name,variant', MODES)
def test_ragged_stream_shapes_and_resolution(cuda_device, mode_name, variant, dist):
    """W < 64, items starting mid-row, partial last slots, last items of 1 and 2 slots, and an odd width (12 x 33) whose
    rows wrap inside pixel pairs (uB == W).  Rows 2..5 of that image carry confidence 1 + 1e-4."""
    out = _ragged_out(RAGGED, RAGGED_EDGES)
    for side, key in ((0, 'pred1'), (1, 'pred2')):
        for e, edge in enumerate(RAGGED_EDGES):
            if edge[side] == 5:
                out[key]['conf'][e][2:6] = 1 + 1e-4 * (1 + torch.rand((4, 33), generator=torch.Generator().manual_seed(e)))
    net = _make(mode_name, out, _params(out, variant, 9), cuda_device, dist=dist, kernel='stream', allow_pw_adaptors=True,
                optimize_pp=True)
    eng = _engine(net)
    from dust3r_b200.cloud_opt.engine import ITEM
    items = eng._items.cpu().numpy().view(ITEM)
    assert {1, 2} <= set(items['nslots'].tolist()), 'items of 1 and 2 slots'
    assert (items['u0'] != 0).any(), 'items that start mid-row'
    assert (items['npx'] < 64 * items['nslots']).any() and any(a % 64 for a in eng.areas), 'partial last slots'
    assert any(w < 64 for h, w in RAGGED) and any(w % 2 for h, w in RAGGED), 'W < 64 and rows that wrap inside a pixel pair'
    check_bounds(eng, f'ragged stream {variant} {dist}', demo_img=5)


@pytest.mark.parametrize('mode_name,variant', MODES)
def test_odd_shapes_general_kernel(cuda_device, mode_name, variant):
    """Odd P, chunk tails, and one image larger than d3r_align_chunk_pixels() and not a multiple of it (45 x 101)."""
    shapes = [(5, 7), (9, 3), (6, 6), (45, 101)]
    edges = [(1, 0), (2, 0), (2, 1), (3, 0), (3, 2), (1, 3)]
    out = _ragged_out(shapes, edges, seed=5)
    net = _make(mode_name, out, _params(out, variant, 4), cuda_device, allow_pw_adaptors=True, optimize_pp=True)
    eng = _engine(net)
    assert eng.kernel == 'general' and 45 * 101 > _lib.get_lib().d3r_align_chunk_pixels()
    assert eng.n_chunks > len(shapes)
    check_bounds(eng, f'odd general {variant}')


@pytest.mark.parametrize('kernel', KERNELS)
def test_leaf_image_next_to_high_degree_images(cuda_device, kernel):
    n, H, W = 6, 16, 32
    edges = _edges(5) + [(5, 0)]
    out = synth_pair_predictions(n, edges, H, W, seed=6)
    net = _make('PointCloudOptimizer', out, _params(out, 'stacked', 3), cuda_device, kernel=kernel)
    check_bounds(_engine(net), f'leaf {kernel}')


def test_mixed_degrees_around_the_entry_window(cuda_device):
    """Images whose degree is exactly the entry window Wn (a full window, no spill), Wn + 1 (a second window of one
    entry), Wn + 2, and 2 or 3, in one item table: m = Wn/2 + 1 views fully connected both ways plus two images attached
    to a few of them."""
    Wn = int(_lib.get_lib().d3r_align_stream_max_window())
    assert Wn % 2 == 0
    m = Wn // 2 + 1                      # degree 2 (m - 1) = Wn inside the clique
    n, H, W = m + 2, 8, 16
    edges = _edges(m) + [(m, 0), (m + 1, 1), (2, m + 1), (3, m), (m, 3)]
    out = synth_pair_predictions(n, edges, H, W, seed=8)
    net = _make('PointCloudOptimizer', out, _params(out, 'stacked', 4, away_from_zero=False), cuda_device, kernel='stream')
    eng = _engine(net)
    deg = set(np.diff(eng._ent_ptr.cpu().numpy()).tolist())
    assert eng.stream_window == Wn and {Wn, Wn + 1, Wn + 2, 2, 3} <= deg, (Wn, deg)
    check_bounds(eng, f'mixed degrees around Wn={Wn} stream')


@pytest.mark.parametrize('conf', ['log', 'm1', 'sqrt', 'id'])
@pytest.mark.parametrize('kernel', KERNELS)
def test_zero_weight_pixels_and_conf_transforms(cuda_device, conf, kernel):
    """Raw confidence exactly 1.0 on a quarter of the pixels: w = 0 terms with 'log' and 'm1'."""
    n, H, W = 3, 16, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=12)
    out['pred1']['conf'][:, :4] = 1.0
    out['pred2']['conf'][:, :, :8] = 1.0
    net = _make('PointCloudOptimizer', out, _params(out, 'stacked', 7, away_from_zero=False), cuda_device, conf=conf, kernel=kernel)
    check_bounds(_engine(net), f'conf {conf} {kernel}')


@pytest.mark.parametrize('kernel', KERNELS)
def test_fx_and_fy_and_presets(cuda_device, kernel):
    """Both focal slots free; then preset poses on two Modular images (norm_pw_scale off) and a preset focal."""
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=11)
    P0 = _params(out, 'per_edge', 6, fx_and_fy=True)
    P0['im_focals'] = P0['im_focals'] + torch.tensor([[0.3, -0.2]])
    net = _make('ModularPointCloudOptimizer', out, P0, cuda_device, fx_and_fy=True, kernel=kernel)
    eng = _engine(net)
    assert not eng.tied_focal
    check_bounds(eng, f'fx_and_fy {kernel}')
    net = _make('ModularPointCloudOptimizer', out, _params(out, 'per_edge', 2), cuda_device, kernel=kernel)
    poses = [torch.eye(4) for _ in range(2)]
    poses[1][:3, 3] = torch.tensor([0.3, 0.0, 0.1])
    net.preset_pose(poses, [0, 1])
    net.preset_focal([40.0], [2])
    eng = _engine(net)
    assert not eng.norm_pw_scale
    check_bounds(eng, f'presets {kernel}')


def test_config3_full_size(cuda_device):
    """BASELINE config 3 at full size: 8 views, 28 pairs, 512x384, PointCloudOptimizer, streaming kernel."""
    n, H, W = 8, 384, 512
    out = synth_pair_predictions(n, _edges(n, symmetrize=False), H, W, seed=0)
    net = _make('PointCloudOptimizer', out, init_params(AlignProblem.from_output(out), seed=0), cuda_device)
    eng = _engine(net)
    assert eng.kernel == 'stream'
    check_adam_step(eng, 1, 'config3 full size')


@pytest.mark.parametrize('kernel', KERNELS)
def test_config5_graph_fixed_point_share(cuda_device, kernel):
    """BASELINE config 5's graph (50 views, 1225 pairs, Modular, coefficients 1 / (P E)) at 64x80."""
    n, H, W = 50, 64, 80
    out = synth_pair_predictions(n, _edges(n, symmetrize=False), H, W, seed=2)
    net = _make('ModularPointCloudOptimizer', out, init_params(AlignProblem.from_output(out, variant='per_edge'), seed=3),
                cuda_device, kernel=kernel)
    eng = _engine(net)
    assert eng.E == 1225
    rep = check_bounds(eng, f'config5 {kernel}')
    print(f'[config5 {kernel}] fixed-point share of the small-gradient bound: max {rep["fixed_point_share_max"]:.3g}, '
          f'median {rep["fixed_point_share_median"]:.3g}')


# ------------------------------------------------------------------------------------------ the Adam step
def check_adam_step(eng, k, label, niter=8):
    """Iterations [0, k) of a schedule of `niter`, a snapshot, the gradient launch at that state (its bounds checked
    as above), then iteration k; every element of logd / exp_avg / exp_avg_sq and of the trainable small parameters and
    their moments against oracle.align_float64.adam64 from the snapshot, the exported gradient and the fp32 sched row.
    The gradient launch re-derives the transforms from `small` (prepare), so iteration k reads the same transforms."""
    lib, dev = eng.lib, eng.device
    eng.reset_adam()
    eng.sched = torch.from_numpy(eng.make_schedule(niter, 0.01)).to(dev)
    eng.loss_out = torch.zeros((niter,), dtype=torch.float32, device=dev)
    eng.prepare()
    if k > 0:
        eng._call(lib.d3r_align_run, C.byref(eng._desc()), 0, k)
    names = ('logd', 'logd_m', 'logd_v', 'small', 'small_m', 'small_v')
    snap = {nm: getattr(eng, nm).detach().clone() for nm in names}
    grads = {}
    check_bounds(eng, f'{label}, state before step {k}', grads=grads)
    eng._call(lib.d3r_align_run, C.byref(eng._desc()), k, k + 1)
    after = {nm: getattr(eng, nm).detach().clone() for nm in names}
    assert torch.isfinite(eng.loss_out[k])
    row = eng.sched[k].double().cpu()
    step_size, bc2s = float(row[1]), float(row[2])
    d = lambda t: t.double().cpu()
    rep = {}
    # per pixel: the exported gradient is the iteration's own (asserted bit for bit at k = 0)
    pix = torch.zeros(int(eng.pix_off[-1]), dtype=torch.bool)
    for i in range(eng.n):
        pix[int(eng.pix_off[i]):int(eng.pix_off[i]) + eng.areas[i]] = True
    g = d(grads['logd'])[pix]
    p1, m1, v1, ep, em, ev = A.adam64(d(snap['logd'])[pix], d(snap['logd_m'])[pix], d(snap['logd_v'])[pix], g, step_size, bc2s,
                                      approx=eng.kernel == 'stream')
    rep['logd'] = A.ratio((d(after['logd'])[pix] - p1).abs(), ep)
    rep['logd_m'] = A.ratio((d(after['logd_m'])[pix] - m1).abs(), em)
    rep['logd_v'] = A.ratio((d(after['logd_v'])[pix] - v1).abs(), ev)
    for nm in ('logd', 'logd_m', 'logd_v'):
        assert torch.equal(after[nm].cpu()[~pix], snap[nm].cpu()[~pix]), f'padding pixels of {nm} must be bit-unchanged'
    if k == 0:
        # zero moments: exp_avg = fl(0.1f * gd), exp_avg_sq = fl(exp_avg * gd), one rounding each, so both must equal
        # what the exported gradient gives bit for bit -- the gradient launch and the iteration compute the same gd
        g32 = grads['logd'].cpu().numpy()[pix.numpy()]
        c1 = np.float32(1) - np.float32(0.9)
        m_want = (np.float64(c1) * g32.astype(np.float64)).astype(np.float32)
        v_want = (m_want.astype(np.float64) * g32.astype(np.float64)).astype(np.float32)
        assert np.array_equal(after['logd_m'].cpu().numpy()[pix.numpy()], m_want)
        assert np.array_equal(after['logd_v'].cpu().numpy()[pix.numpy()], v_want)
    # small parameters: the iteration's own sums may differ from the exported ones (odd iterations walk the items in
    # reverse), both are within the small-gradient bound of float64, hence dg = 2 * bound
    tr = eng.small_trainable.cpu().bool()
    p1, m1, v1, ep, em, ev = A.adam64(d(snap['small'])[tr], d(snap['small_m'])[tr], d(snap['small_v'])[tr], d(grads['small'])[tr],
                                      step_size, bc2s, approx=False, dg=2 * grads['small_bound'][tr])
    rep['small'] = A.ratio((d(after['small'])[tr] - p1).abs(), ep)
    rep['small_m'] = A.ratio((d(after['small_m'])[tr] - m1).abs(), em)
    rep['small_v'] = A.ratio((d(after['small_v'])[tr] - v1).abs(), ev)
    for nm in ('small', 'small_m', 'small_v'):
        assert torch.equal(after[nm].cpu()[~tr], snap[nm].cpu()[~tr]), f'non-trainable entries of {nm} must be bit-unchanged'
        if eng.tied_focal:
            o = eng._offsets()
            f = after[nm][o['focals']:o['pp']].reshape(eng.n, 2)
            assert torch.equal(f[:, 0], f[:, 1]), f'tied focals of {nm} must stay equal'
    assert (~tr).any() and tr.any()
    print(f'[{label}] Adam step {k} worst err/bound: ' + ', '.join(f'{kk}={v:.3g}' for kk, v in rep.items()))
    for kk, v in rep.items():
        assert v <= 1.0, (label, k, kk, rep)
    return rep


ADAM_SHAPES = [(24, 32), (20, 36), (12, 33), (16, 20)]
ADAM_EDGES = [(1, 0), (2, 0), (2, 1), (0, 2), (3, 1), (0, 3), (3, 2)]


@pytest.mark.parametrize('k', [0, 3, 4])
@pytest.mark.parametrize('mode_name,dist', [('PointCloudOptimizer', 'l1'), ('ModularPointCloudOptimizer', 'l2')])
@pytest.mark.parametrize('kernel', KERNELS)
def test_adam_step_element_by_element(cuda_device, kernel, mode_name, dist, k):
    """Ragged shapes (padded stacked depth), principal points and adaptors not trainable, tied focals; k = 0 (zero
    moments, bit identity of the exported and the iteration's gd), k = 3 (odd: the streaming kernel walks items_rev)
    and k = 4."""
    out = _ragged_out(ADAM_SHAPES, ADAM_EDGES, seed=13)
    variant = 'stacked' if mode_name == 'PointCloudOptimizer' else 'per_edge'
    net = _make(mode_name, out, _params(out, variant, 11), cuda_device, dist=dist, kernel=kernel)
    eng = _engine(net)
    assert eng.kernel == kernel and eng.tied_focal
    if kernel == 'stream':
        assert eng._items_rev is not None
    check_adam_step(eng, k, f'adam {kernel} {variant} {dist}')


# ------------------------------------------------------------------------------------------ packing and world points
CONF_MODES = {'id': lambda c: c, 'm1': lambda c: c - np.float32(1), 'log': np.log, 'sqrt': np.sqrt}


@pytest.mark.parametrize('conf', list(CONF_MODES))
@pytest.mark.parametrize('kernel', KERNELS)
def test_pack_entries_against_numpy(cuda_device, conf, kernel):
    from dust3r_b200.cloud_opt.engine import AlignEngine
    shapes = [(24, 32), (12, 33), (20, 36)] if kernel == 'stream' else [(5, 7), (9, 3), (20, 36)]
    edges = [(1, 0), (2, 0), (2, 1), (0, 2)]
    out = _ragged_out(shapes, edges, seed=7)
    pi, pj = out['pred1']['pts3d'], out['pred2']['pts3d_in_other_view']
    ci, cj = out['pred1']['conf'], out['pred2']['conf']
    eng = AlignEngine(edges, shapes, pi, pj, ci, cj, cuda_device, conf_mode=conf, kernel=kernel)
    obs = eng.obs.cpu().numpy()
    off = eng._ent_obs_off.cpu().numpy()
    coef = eng._ent_coef.cpu().numpy()
    edge_ent = eng._edge_ent.cpu().numpy()
    used = np.zeros(len(obs), dtype=bool)
    for e, (i, j) in enumerate(edges):
        for side, img, pts, cf in ((0, i, pi[e], ci[e]), (1, j, pj[e], cj[e])):
            k = edge_ent[e, side]
            P = shapes[img][0] * shapes[img][1]
            q = pts.reshape(-1, 3).numpy()
            c = cf.reshape(-1).numpy()
            trf32 = CONF_MODES[conf](c).astype(np.float32)
            trf64 = CONF_MODES[conf](c.astype(np.float64))
            o = int(off[k])
            if kernel == 'stream':
                ns = (P + 63) // 64
                slab = obs[o:o + 64 * ns].reshape(ns, 2, 32, 4)
                x, y = slab[:, 0, :, 0:2].reshape(-1), slab[:, 0, :, 2:4].reshape(-1)
                z, w = slab[:, 1, :, 0:2].reshape(-1), slab[:, 1, :, 2:4].reshape(-1)
                used[o:o + 64 * ns] = True
                assert not x[P:].any() and not y[P:].any() and not z[P:].any() and not w[P:].any(), 'padding must be 0.0'
                w_ref32, w_ref64 = np.float32(coef[k]) * trf32, np.float64(coef[k]) * trf64
                ulps = 2
            else:
                x, y, z, w = obs[o:o + P].T
                used[o:o + P] = True
                w_ref32, w_ref64 = trf32, trf64
                ulps = 1
            assert np.array_equal(np.stack((x[:P], y[:P], z[:P]), -1), q), 'positions are copied bit for bit'
            if conf in ('id', 'm1'):
                assert np.array_equal(w[:P], w_ref32)
            else:
                assert np.all(np.abs(w[:P].astype(np.float64) - w_ref64) <= ulps * np.spacing(np.abs(w_ref32)))
    assert used.all(), 'every slab sits where ent_obs_off says, and the slabs tile the buffer'


@pytest.mark.parametrize('shapes', [[(24, 32), (20, 36), (14, 44), (12, 33)], [(5, 7), (9, 3), (45, 101)]])
def test_pts3d_against_float64(cuda_device, shapes):
    edges = [(1, 0), (2, 0), (2, 1), (0, 2)] + ([(3, 1)] if len(shapes) > 3 else [])
    out = _ragged_out(shapes, edges, seed=2)
    net = _make('ModularPointCloudOptimizer', out, _params(out, 'per_edge', 8), cuda_device)
    eng = _engine(net)
    X = eng.pts3d().double().cpu()
    sc = A.scene_from_engine(eng)
    geo = A.image_geometry(sc, sc.small, sc.logd)
    worst = 0.0
    for i, g in enumerate(geo):
        a, P = int(eng.pix_off[i]), eng.areas[i]
        bound = A.C3 * A.U * ((g['Cm'] @ g['R'].abs().T).sum(-1) + g['T'].abs().sum()) + 2 * 2.0 ** -23 * g['Y'].abs().sum(-1)
        worst = max(worst, A.ratio((X[a:a + P] - g['X']).abs().max(-1).values, bound))
    print(f'\n[pts3d {shapes}] worst err/bound {worst:.3g}')
    assert worst <= 1


# ------------------------------------------------------------------------------------------ overflow and NaN contract
def _overflow_scene(cuda_device, kernel, how):
    n, H, W = 4, 24, 32
    scale = {'nan': 1.0, 'huge': 1e4, 'in_range': 100.0}[how]
    out = _ragged_out([(H, W)] * n, _edges(n), seed=1, scale=scale)
    if how == 'nan':
        out['pred1']['pts3d'][2][5, 7, 1] = float('nan')
    P0 = _params(out, 'per_edge', 5)
    return out, P0, dict(dist='l2' if how != 'nan' else 'l1', kernel=kernel)


@pytest.mark.parametrize('how', ['nan', 'huge'])
@pytest.mark.parametrize('mode_name,variant', MODES)
@pytest.mark.parametrize('kernel', KERNELS)
def test_out_of_range_scene_is_never_finite_and_silent(cuda_device, kernel, mode_name, variant, how):
    out, P0, kw = _overflow_scene(cuda_device, kernel, how)
    net = _make(mode_name, out, P0, cuda_device, **kw)
    with pytest.raises(_lib.D3RError):
        net.compute_global_alignment(init=None, niter=3)
    net = _make(mode_name, out, P0, cuda_device, **kw)
    with torch.no_grad():
        assert torch.isnan(net())
    loss = net()
    assert torch.isnan(loss.detach())
    loss.backward()
    assert torch.isnan(net.pw_poses.grad).all()
    if mode_name == 'ModularPointCloudOptimizer':
        loss, details = net(ret_details=True)
        on = details != -1
        assert torch.isnan(loss.detach()) and torch.isnan(details[on]).all()
        assert all(torch.isnan(p.grad).all() for p in net.im_poses if p.grad is not None)
    else:
        assert torch.isnan(net.im_poses.grad).all() and torch.isnan(net.im_focals.grad).all()


@pytest.mark.parametrize('kernel', KERNELS)
def test_flag_clears_after_an_overflowing_call(cuda_device, kernel):
    n, H, W = 4, 24, 32
    out = synth_pair_predictions(n, _edges(n), H, W, seed=1)
    net = _make('PointCloudOptimizer', out, _params(out, 'stacked', 5), cuda_device, kernel=kernel)
    eng = _engine(net)
    loss0, _, g0, _ = eng.loss_and_grad()
    eng.check_overflow()
    saved = eng.obs[17].clone()
    eng.obs[17, 0] = float('nan')
    loss, _, g, _ = eng.loss_and_grad()
    assert torch.isnan(loss) and torch.isnan(g).all()
    with pytest.raises(_lib.D3RError):
        eng.check_overflow()
    eng.obs[17] = saved
    loss, _, g, _ = eng.loss_and_grad()
    eng.check_overflow()
    assert torch.equal(loss, loss0) and torch.equal(g, g0)


@pytest.mark.parametrize('kernel', KERNELS)
def test_in_range_scaled_scene_passes_the_bounds(cuda_device, kernel):
    """Pointmaps x100 with l2: partial sums stay inside the fixed-point range, nothing is raised, every element is
    within the float64 bounds."""
    out, P0, kw = _overflow_scene(cuda_device, kernel, 'in_range')
    net = _make('PointCloudOptimizer', out, P0, cuda_device, **kw)
    check_bounds(_engine(net), f'x100 l2 {kernel}')
    net.compute_global_alignment(init=None, niter=3)
    assert torch.isfinite(net.last_losses).all()
