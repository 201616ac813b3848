"""The float64 alignment oracle (oracle/align_float64.py) on the CPU: its vectorised per-pixel gradient and its loss equal
autograd of the reference objective (oracle.align_oracle.loss_fn) run in float64, and the element-wise bounds it builds
see the three kernel mistakes tests/test_align_float64_gpu.py demonstrates (a pixel unprojected one column off at a row
wrap, one entry dropped from one pixel, one pixel missing from one entry's sums)."""
import numpy as np
import pytest
import torch

from dust3r_b200.cloud_opt.engine import build_stream_items, SLOT_PX
from oracle import align_float64 as A
from oracle.align_oracle import AlignProblem, init_params, loss_fn

SHAPES = [(8, 12), (6, 10), (4, 15)]          # 4 x 15: odd width, rows wrap inside pixel pairs
EDGES = [(1, 0), (2, 0), (2, 1), (0, 2), (0, 1)]


def _problem(dist, variant, seed=0, fx_and_fy=False):
    g = torch.Generator().manual_seed(seed)
    p1 = [torch.randn(SHAPES[i] + (3,), generator=g, dtype=torch.float64) + torch.tensor([0, 0, 3.], dtype=torch.float64) for i, j in EDGES]
    p2 = [torch.randn(SHAPES[j] + (3,), generator=g, dtype=torch.float64) + torch.tensor([0, 0, 3.], dtype=torch.float64) for i, j in EDGES]
    c1 = [1 + 5 * torch.rand(SHAPES[i], generator=g, dtype=torch.float64) for i, j in EDGES]
    c2 = [1 + 5 * torch.rand(SHAPES[j], generator=g, dtype=torch.float64) for i, j in EDGES]
    out = dict(view1=dict(idx=[i for i, j in EDGES]), view2=dict(idx=[j for i, j in EDGES]),
               pred1=dict(pts3d=p1, conf=c1), pred2=dict(pts3d_in_other_view=p2, conf=c2))
    prob = AlignProblem.from_output(out, dist=dist, variant=variant)
    prob.pred_i = [x.reshape(-1, 3) for x in p1]
    prob.pred_j = [x.reshape(-1, 3) for x in p2]
    prob.weight_i = [x.reshape(-1).log() for x in c1]
    prob.weight_j = [x.reshape(-1).log() for x in c2]
    P = init_params(prob, seed=seed + 1, fx_and_fy=fx_and_fy)
    P = {k: ([t.double() for t in v] if isinstance(v, list) else v.double()) for k, v in P.items()}
    P['pw_adaptors'] = 0.5 * torch.randn(P['pw_adaptors'].shape, generator=g, dtype=torch.float64)
    P['im_pp'] = 0.3 * torch.randn(P['im_pp'].shape, generator=g, dtype=torch.float64)
    if fx_and_fy:
        P['im_focals'] = P['im_focals'] + torch.tensor([[0.3, -0.2]], dtype=torch.float64)
    return prob, P


def _stream_chains(sc):
    areas = [h * w for h, w in sc.imshapes]
    deg = np.bincount(sc.ent_img, minlength=sc.n)
    ent_ptr = np.concatenate([[0], np.cumsum(deg)])
    slots = [(a + SLOT_PX - 1) // SLOT_PX for a in areas]
    ent_off = np.concatenate([[0], np.cumsum([slots[i] * SLOT_PX for i in sc.ent_img])])[:-1]
    pix_off = np.concatenate([[0], np.cumsum(areas)])
    items, warp_ptr, _ = build_stream_items(sc.imshapes, pix_off, ent_ptr, ent_off, slots, 3, 8, 4)
    return dict(items=items, warp_ptr=warp_ptr, window=int(deg.max()))


def _autograd(prob, P):
    Q = {k: ([t.clone().requires_grad_(True) for t in v] if isinstance(v, list) else v.clone().requires_grad_(True))
         for k, v in P.items()}
    loss = loss_fn(prob, Q)
    loss.backward()
    return float(loss.detach()), {k: ([t.grad for t in v] if isinstance(v, list) else v.grad) for k, v in Q.items()}


@pytest.mark.parametrize('fx_and_fy', [False, True])
@pytest.mark.parametrize('dist', ['l1', 'l2'])
@pytest.mark.parametrize('variant', ['stacked', 'per_edge'])
def test_oracle_matches_float64_autograd(variant, dist, fx_and_fy):
    prob, P = _problem(dist, variant, fx_and_fy=fx_and_fy)
    l_ref, g_ref = _autograd(prob, P)
    sc = A.scene_from_problem(prob, P, fx_and_fy=fx_and_fy)
    T = A.terms(sc)
    for i in range(sc.n):
        scale = float(g_ref['im_depthmaps'][i].abs().max())
        assert float((T['gd'][i] - g_ref['im_depthmaps'][i]).abs().max()) <= 1e-12 * scale
    L, _, l_tot, _ = A.loss_bounds(sc, _chained(sc))
    assert abs(l_tot - l_ref) <= 1e-12 * abs(l_ref)
    l64, g = A.small_grad64(sc)
    assert abs(l64 - l_ref) <= 1e-12 * abs(l_ref)
    o = sc.offsets()
    n, E = sc.n, sc.E
    want = dict(poses=g_ref['im_poses'].reshape(-1), pp=g_ref['im_pp'].reshape(-1), pw=g_ref['pw_poses'].reshape(-1),
                adapt=g_ref['pw_adaptors'].reshape(-1))
    got = dict(poses=g[o['poses']:o['focals']], pp=g[o['pp']:o['pw']], pw=g[o['pw']:o['adapt']], adapt=g[o['adapt']:])
    for k in want:
        assert torch.allclose(got[k], want[k], rtol=1e-12, atol=1e-12 * float(want[k].abs().max())), k
    gf = g[o['focals']:o['pp']].reshape(n, 2)
    wf = g_ref['im_focals'].reshape(n, -1)
    if fx_and_fy:
        assert torch.allclose(gf, wf, rtol=1e-12, atol=0)
    else:
        assert torch.allclose(gf[:, 0], wf[:, 0], rtol=1e-12, atol=0) and torch.equal(gf[:, 0], gf[:, 1])


def _chained(sc):
    A.set_chains(sc, **_stream_chains(sc))
    return A.terms(sc)


def test_entry_order_is_the_engine_csr():
    img, edge, side = A.entry_order(3, EDGES)
    assert img.tolist() == [0, 0, 0, 0, 1, 1, 1, 2, 2, 2]
    assert [(e, s) for e, s in zip(edge, side)][:4] == [(0, 1), (1, 1), (3, 0), (4, 0)]


@pytest.mark.parametrize('dist', ['l1', 'l2'])
def test_resolution_checks_trip_on_the_oracles_perturbations(dist):
    """Each mutation exceeds the element-wise bound where it lands (ratio > 1)."""
    prob, P = _problem(dist, 'stacked', seed=4)
    sc = A.scene_from_problem(prob, P)
    T = _chained(sc)
    sb, _ = A.small_bound(sc, T)
    _, g = A.small_grad64(sc)
    demo = A.resolution_demo(sc, T, sb, g)
    print(demo)
    for name, res in demo.items():
        assert res is not None and res[0] > 1, (name, res)


def test_small_bound_covers_fp32_parameters():
    """The bound is no tautology: rounding the parameters to fp32 moves the float64 gradient by far less than it allows,
    and a 1e-3 relative change of one log-scale moves it by more."""
    prob, P = _problem('l1', 'stacked', seed=2)
    sc = A.scene_from_problem(prob, P)
    T = _chained(sc)
    sb, fixed = A.small_bound(sc, T)
    assert bool((fixed <= sb).all()) and bool((sb > 0).all())
    _, g = A.small_grad64(sc)
    sc32 = A.scene_from_problem(prob, {k: ([t.float().double() for t in v] if isinstance(v, list) else v.float().double())
                                       for k, v in P.items()})
    _, g32 = A.small_grad64(sc32)
    assert A.ratio((g32 - g).abs(), sb) < 1
    sc2 = A.scene_from_problem(prob, P)
    sc2.small = sc2.small.clone()
    sc2.small[sc.offsets()['pw'] + 7] *= 1.001
    _, g2 = A.small_grad64(sc2)
    assert A.ratio((g2 - g).abs(), sb) > 1
