"""The float64 scene oracle (oracle/scene_float64.py) on the CPU: it equals the unmodified reference run in float64 (clean
decisions, Weiszfeld focals, nearest neighbours; tests/golden/scene_ops.npz) and the host ports run in float64; the reference's
fp32 outputs agree with it on every decided pixel and lie within its fp32 focal bound; and the comparison helpers the GPU test
uses flag deliberate kernel mistakes (the resolution demonstration): half away from zero, `<=` in the depth test, parallel
semantics and image i's width in the clean filter; a dropped point and the previous problem's weights in the Procrustes
moments; one iteration fewer, a 1e-6 clip and NaN rays kept in the Weiszfeld focal; the highest index on ties and a skipped
last point of a tile in the nearest neighbours.

The inputs are generated here from seeds (tests/test_scene_float64_gpu.py runs the same ones on the device); the golden
holds the reference's outputs only (tests/golden/make_scene_golden.py)."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import scene_float64 as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'scene_ops.npz')
KTILE = 2048                      # points per shared-memory tile of nn_kernel (kTile in scene_ops.cu)


# ------------------------------------------------------------------------------------------------------------ inputs
def _rot_y(a):
    return torch.tensor([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]], dtype=torch.float64)


def clean_scene(shapes, seed, extras=False, spread=0.2):
    """Cameras on an arc looking at one rough surface, one image per shape: dict(pts [(H,W,3)], conf [(H,W)], depth [(H,W)],
    K (n,3,3), T (n,4,4) world -> camera), fp32.  extras: points behind every camera, points off every image, NaN points and
    NaN depths."""
    g = torch.Generator().manual_seed(seed)
    n = len(shapes)
    out = dict(pts=[], conf=[], depth=[], K=[], T=[])
    for i, (H, W) in enumerate(shapes):
        f = 1.1 * max(H, W)
        K = torch.tensor([[f, 0, W / 2 + 0.25], [0, f, H / 2 - 0.25], [0, 0, 1]], dtype=torch.float64)
        ang = spread * (i - (n - 1) / 2)
        c2w = torch.eye(4, dtype=torch.float64)
        c2w[:3, :3] = _rot_y(ang)
        c2w[:3, 3] = torch.tensor([0.8 * math.sin(ang), 0.03 * i, 0.1 * (1 - math.cos(ang))])
        vs, us = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing='ij')
        d = 2.0 + torch.nn.functional.interpolate(torch.rand((1, 1, 5, 5), generator=g, dtype=torch.float64), size=(H, W),
                                                  mode='bicubic', align_corners=True)[0, 0]
        d = d + 0.3 * torch.rand((H, W), generator=g, dtype=torch.float64)
        cam = torch.stack(((us - K[0, 2]) * d / f, (vs - K[1, 2]) * d / f, d), -1)
        pts = cam @ c2w[:3, :3].T + c2w[:3, 3]
        conf = 1 + 3 * torch.rand((H, W), generator=g, dtype=torch.float64)
        if extras:
            m = torch.rand((H, W), generator=g) < 0.03
            pts[m] = pts[m] * torch.tensor([1.0, 1.0, -1.0], dtype=torch.float64) - torch.tensor([0, 0, 3.0], dtype=torch.float64)
            m = torch.rand((H, W), generator=g) < 0.03
            pts[m] = pts[m] + torch.tensor([40.0, -25.0, 0.0], dtype=torch.float64)
            pts[torch.rand((H, W), generator=g) < 0.01] = float('nan')
            d[torch.rand((H, W), generator=g) < 0.01] = float('nan')
        out['pts'].append(pts.float())
        out['conf'].append(conf.float())
        out['depth'].append(d.float())
        out['K'].append(K.float())
        out['T'].append(torch.linalg.inv(c2w).float())
    out['K'], out['T'] = torch.stack(out['K']), torch.stack(out['T'])
    return out


def half_scene():
    """Identity cameras (K = I, T = I): image 0's points project exactly onto u = k + 0.5 and v = l + 0.5 (and exactly onto
    integers), so rintf's half to even picks the pixel; some points sit exactly at image 1's depth (tol = 0 decides `<`)."""
    H, W = 6, 8
    vs, us = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing='ij')
    z = torch.ones((H, W))
    pts0 = torch.stack((us + 0.5 * (us.long() % 2 == 0), vs + 0.5 * (vs.long() % 3 == 0), z), -1)
    pts0 = pts0 * torch.where(us.long() % 4 == 1, 2.0, 1.0)[..., None]       # exact scaling by 2: still exact quotients
    pts1 = torch.stack((us, vs, torch.full((H, W), 3.0)), -1)
    depth0 = pts0[..., 2].clone()
    depth1 = torch.where((us + vs).long() % 2 == 0, torch.full((H, W), 2.0), torch.full((H, W), 1.0))   # 1 or 2: at or behind
    conf0 = 1 + (us + 2 * vs) % 5 * 0.5
    conf1 = 4 - (2 * us + vs) % 7 * 0.4
    eye = torch.eye(4)
    return dict(pts=[pts0, pts1], conf=[conf0, conf1], depth=[depth0, depth1], K=torch.eye(3).repeat(2, 1, 1),
                T=eye.repeat(2, 1, 1))


def chain_scene(n=3, H=24, W=32, seed=7):
    """Cameras 0 .. n-2 identical (image i's pixel p lands on pixel p of the others, at its own depth), camera n-1 shifted
    sideways by 4 / depth pixels, so that it sees images 0 and 1 at different pixels.  Random depths and confidences then make
    chains where image 0's cut (by image n-1) decides whether image 1 is cut by image 0: sequential and parallel semantics
    differ."""
    g = torch.Generator().manual_seed(seed)
    f = 40.0
    K = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]])
    vs, us = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing='ij')
    pts, conf, depth = [], [], []
    for i in range(n):
        d = 1 + torch.randint(0, 4, (H, W), generator=g).to(torch.float64)
        pts.append(torch.stack(((us - W / 2) * d / f, (vs - H / 2) * d / f, d), -1).float())
        depth.append(d.float())
        conf.append(1 + torch.randint(0, 7, (H, W), generator=g).float() * 0.5)
    T = torch.eye(4).repeat(n, 1, 1)
    T[-1, 0, 3] = 0.1
    return dict(pts=pts, conf=conf, depth=depth, K=K.repeat(n, 1, 1), T=T)


def clean_cases():
    """name -> (scene, tol, bad_conf)."""
    mixed = [(48, 64), (64, 48), (37, 53), (48, 64), (37, 53)]
    return {
        'n1': (clean_scene([(37, 53)], 1), 0.001, 0.0),
        'n2_mixed': (clean_scene(mixed[1:3], 2, extras=True), 0.001, 0.0),
        'n5_mixed_tol0': (clean_scene(mixed, 3, extras=True), 0.0, 0.0),
        'n5_mixed_tol0.3_bad1.5': (clean_scene(mixed, 4, extras=True), 0.3, 1.5),
        'n5_same_tol0.001_bad1.5': (clean_scene([(48, 64)] * 5, 5), 0.001, 1.5),
        'half': (half_scene(), 0.0, 0.0),
        'chain': (chain_scene(), 0.001, 0.0),
    }


def flat(scene):
    """The oracle's view of a scene: flat fp32 per-image arrays, the shapes, K and T."""
    hw = [tuple(c.shape) for c in scene['conf']]
    return ([p.reshape(-1, 3) for p in scene['pts']], [c.reshape(-1) for c in scene['conf']],
            [d.reshape(-1) for d in scene['depth']], hw, scene['K'], scene['T'])


def weiszfeld_maps(H, W, seed, B=4, degenerate=True):
    """B camera-frame pointmaps with different focals and off-centre principal points (map 0's is integer, the others are not):
    (pts (B,H,W,3), pp (B,2)) fp32.  degenerate: a 0/0 pixel, x/0 = +-inf, a NaN point, and on map 0 a zero ray at the principal
    point (residual 0 there: the 1e-8 clip applies)."""
    g = torch.Generator().manual_seed(seed)
    vs, us = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing='ij')
    pts, pps = [], []
    for b in range(B):
        f = [90.0, 140.0, 210.0, 333.0][b % 4] * max(H, W) / 128
        pp = torch.tensor([W // 2 - 1, H // 2], dtype=torch.float64) if b == 0 else \
            torch.tensor([W / 2 + 0.37 * b, H / 2 - 0.21 * b], dtype=torch.float64)
        d = 1.5 + torch.rand((H, W), generator=g, dtype=torch.float64)
        p = torch.stack(((us - pp[0]) * d / f, (vs - pp[1]) * d / f, d), -1)
        p = p + 0.02 * torch.randn(p.shape, generator=g, dtype=torch.float64)
        if degenerate and H * W >= 8:
            flat_p = p.reshape(-1, 3)
            flat_p[1] = torch.tensor([0.0, 0.0, 0.0])
            flat_p[2] = torch.tensor([1.0, -2.0, 0.0])
            flat_p[3] = float('nan')
            if b == 0:
                flat_p[int(pp[1]) * W + int(pp[0])] = torch.tensor([0.0, 0.0, 1.7])
        pts.append(p.float())
        pps.append(pp.float())
    return torch.stack(pts), torch.stack(pps)


def nn_points(M, seed, ties=True):
    """M Gaussian points; with ties: duplicates at 100 and 2148 (both sides of the first tile boundary) when M allows."""
    g = torch.Generator().manual_seed(seed)
    p = torch.randn((M, 3), generator=g)
    if ties and M > 2148:
        p[2148] = p[100]
    return p


def nn_queries(N, points, seed):
    """N queries: Gaussian, plus exact copies of the last point of every tile, of point 0 and of the duplicated point."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn((N, 3), generator=g)
    M = points.shape[0]
    picks = [M - 1, 0] + list(range(KTILE - 1, M, KTILE)) + ([100, 2148] if M > 2148 else [])
    for k, idx in enumerate(picks[:N]):
        q[(k * 37) % N] = points[idx]
    return q


def perm_quat(g):
    q = torch.randn(4, generator=g, dtype=torch.float64)
    w, x, y, z = (q / q.norm()).tolist()
    return torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                         [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                         [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], dtype=torch.float64)


def procrustes_problems(B, P, seed, kind='general'):
    """B problems of P points, each with its own rotation, scale, translation and weights: x, y (B,P,3), w (B,P) fp32.
    kind: 'general', 'planar' (x in a plane), 'mirror' (y a reflection of x: D = -1), 'far' (centre 10^3 x the spread),
    'half_zero' (half the weights 0), 'anchor' (no weights: all ones)."""
    g = torch.Generator().manual_seed(seed)
    xs, ys, ws = [], [], []
    for b in range(B):
        x = torch.randn((P, 3), generator=g, dtype=torch.float64) * torch.tensor([2.0, 1.0, 0.5], dtype=torch.float64)
        if kind == 'planar':
            x[:, 2] = 0.3 * x[:, 0] - 0.2 * x[:, 1] + 1.0
        if kind == 'far':
            x = x + torch.tensor([1500.0, -800.0, 2000.0], dtype=torch.float64)
        R = perm_quat(g)
        if kind == 'mirror':
            R = R @ torch.diag(torch.tensor([1.0, 1.0, -1.0], dtype=torch.float64))
        s = 0.5 + 2 * float(torch.rand(1, generator=g))
        t = torch.randn(3, generator=g, dtype=torch.float64) * 3
        y = s * x @ R.T + t + 0.01 * torch.randn((P, 3), generator=g, dtype=torch.float64)
        w = 0.1 + 5 * torch.rand(P, generator=g, dtype=torch.float64)
        if kind == 'half_zero':
            w[torch.randperm(P, generator=g)[:P // 2]] = 0
        if kind == 'anchor':
            w = torch.ones(P, dtype=torch.float64)
        xs.append(x), ys.append(y), ws.append(w)
    return torch.stack(xs).float(), torch.stack(ys).float(), torch.stack(ws).float()


# ------------------------------------------------------------------------------------------------------- comparison helpers
def moments_ratio(got, m, dm):
    """Largest |got - m| / dm over the 17 moments of every problem (0 where equal)."""
    err = (O.f64(got) - m).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / dm)
    return float(r.max())


def registration_ratios(R, t, s, ref):
    """err / bound of fp32 R, t, s against registration64's result, over the problems whose rotation is unique."""
    ok = ref['gap'] > 0
    out = {}
    for k, v in (('R', R), ('t', t), ('s', s)):
        err = (O.f64(v) - ref[k]).abs()[ok]
        b = ref['d' + k][ok]
        out[k] = float(torch.where(err == 0, torch.zeros_like(err), err / b).max()) if err.numel() else 0.0
    return out, int(ok.sum())


def weiszfeld_chain_ratio(pts, pp, W, focals):
    """focals[k]: the fp32 result of steps = k, k = 0..K.  Largest err / bound of each against one oracle step fed
    focals[k - 1]."""
    B = pts.shape[0]
    P = pts.reshape(B, -1, 3)
    worst = 0.0
    for k, fk in enumerate(focals):
        f, df = O.weiszfeld_step64(P, pp, W, None if k == 0 else focals[k - 1])
        worst = max(worst, O.check_focal(fk, f, df))
    return worst


# ------------------------------------------------------------------------------------------------ the reference (golden)
@pytest.fixture(scope='module')
def golden():
    return dict(np.load(GOLDEN))


GOLDEN_CLEAN = ['n2_mixed', 'n5_mixed_tol0.3_bad1.5', 'n5_same_tol0.001_bad1.5', 'half', 'chain']
GOLDEN_FOCAL = [(5, 7), (33, 31), (48, 64)]
GOLDEN_NN = [(3000, 2500)]


def _as64(scene):
    return {k: ([x.double() for x in v] if isinstance(v, list) else v.double()) for k, v in scene.items()}


@pytest.mark.parametrize('name', GOLDEN_CLEAN)
def test_clean_oracle_equals_reference_float64(name, golden):
    scene, tol, bad = clean_cases()[name]
    pts, conf, depth, hw, K, T = flat(scene)
    res = O.clean64(pts, conf, depth, hw, K, T, tol, bad, coef=1 - tol, u=O.U64)
    for i, (c, und) in enumerate(res):
        assert int(und.sum()) == 0, (name, i, int(und.sum()))
        assert torch.equal(c, torch.from_numpy(golden[f'clean|{name}|f64|{i}']).reshape(-1)), (name, i)


@pytest.mark.parametrize('name', GOLDEN_CLEAN)
def test_clean_oracle_equals_host_port_float64(name):
    from dust3r_b200.cloud_opt.pointcloud_filter import clean_pointcloud
    scene, tol, bad = clean_cases()[name]
    s = _as64(scene)
    got = clean_pointcloud(s['conf'], s['K'], s['T'], s['depth'], s['pts'], tol=tol, bad_conf=bad)
    pts, conf, depth, hw, K, T = flat(scene)
    res = O.clean64(pts, conf, depth, hw, K, T, tol, bad, coef=1 - tol, u=O.U64)
    for (c, und), g in zip(res, got):
        assert not und.any() and torch.equal(c, g.reshape(-1))


@pytest.mark.parametrize('name', GOLDEN_CLEAN)
def test_reference_fp32_clean_agrees_on_decided_pixels(name, golden):
    """The reference's own fp32 evaluation (a different order) agrees with the oracle on every decided pixel, image i against
    the reference's final confidences of images < i."""
    scene, tol, bad = clean_cases()[name]
    pts, conf, depth, hw, K, T = flat(scene)
    ref = [torch.from_numpy(golden[f'clean|{name}|f32|{i}']).reshape(-1) for i in range(len(pts))]
    wrong, und, bad_und, cut = O.check_clean(ref, pts, conf, depth, hw, K, T, tol, bad, coef=float(np.float32(1 - tol)))
    assert wrong == 0 and bad_und == 0, (wrong, bad_und)
    assert cut > 0 and und <= max(2, cut // 50), (und, cut)


def test_half_integer_projections_are_decided():
    scene, tol, bad = clean_cases()['half']
    pts, conf, depth, hw, K, T = flat(scene)
    res = O.clean64(pts, conf, depth, hw, K, T, tol, bad)
    assert not any(bool(u.any()) for _, u in res)
    v = pts[0][:, 0] / pts[0][:, 2]
    assert bool(((v - v.floor()) == 0.5).any())                    # exact halves are present


@pytest.mark.parametrize('shape', GOLDEN_FOCAL)
def test_weiszfeld_oracle_equals_reference(shape, golden):
    H, W = shape
    pts, pp = weiszfeld_maps(H, W, seed=H * W)
    f64 = O.weiszfeld64(pts.reshape(4, -1, 3), pp, W)
    ref64 = torch.from_numpy(golden[f'focal|{H}x{W}|f64'])
    assert torch.allclose(f64, ref64, rtol=1e-12, atol=0), (f64, ref64)
    # the host port in float64
    from dust3r_b200.post_process import estimate_focal_knowing_depth
    port = estimate_focal_knowing_depth(pts.double(), pp.double(), focal_mode='weiszfeld')
    assert torch.allclose(f64, port, rtol=1e-12, atol=0)
    # the reference's fp32 focal, within the fp32-sums bound of the last step fed the host port's fp32 step 9
    from dust3r_b200.post_process import _irls_focal
    from dust3r_b200.utils.geometry import xy_grid
    cpx = xy_grid(W, H, device='cpu').view(1, -1, 2) - pp.view(-1, 1, 2)
    f9 = _irls_focal(cpx, pts.flatten(1, 2), steps=9)
    f, df = O.weiszfeld_step64(pts.reshape(4, -1, 3), pp, W, f9, fp32_sums=True)
    assert O.check_focal(torch.from_numpy(golden[f'focal|{H}x{W}|f32']), f, df) <= 1
    # and every fp32 step of the host port within one oracle step of the previous
    chain = [_irls_focal(cpx, pts.flatten(1, 2), steps=k) for k in range(11)]
    worst = 0.0
    for k, fk in enumerate(chain):
        f, df = O.weiszfeld_step64(pts.reshape(4, -1, 3), pp, W, None if k == 0 else chain[k - 1], fp32_sums=True)
        worst = max(worst, O.check_focal(fk, f, df))
    assert worst <= 1, worst


def test_nn_oracle_equals_reference(golden):
    from dust3r_b200.utils.geometry import find_reciprocal_matches
    for N, M in GOLDEN_NN:
        P1, P2 = nn_points(N, 11, ties=False), nn_points(M, 12, ties=False)
        want = golden[f'nn|{N}x{M}|nn2_in_P1']
        assert np.array_equal(O.nn64(P2, P1).numpy(), want)
        m = golden[f'nn|{N}x{M}|reciprocal_in_P2']
        nn1 = O.nn64(P1, P2)
        assert np.array_equal((nn1[torch.from_numpy(want)] == torch.arange(M)).numpy(), m)
        mp, nnp, cnt = find_reciprocal_matches(P1.numpy(), P2.numpy())
        assert np.array_equal(mp, m) and np.array_equal(nnp, want) and cnt == int(golden[f'nn|{N}x{M}|count'])


def test_registration_oracle_equals_host_port_float64():
    from dust3r_b200.cloud_opt.commons import rigid_points_registration
    for kind in ('general', 'planar', 'mirror', 'far', 'half_zero'):
        x, y, w = procrustes_problems(3, 500, seed=21, kind=kind)
        R, t, s = rigid_points_registration(x.double(), y.double(), weights=w.double(), compute_scaling=True)
        o = O.umeyama64(x, y, w)
        assert torch.allclose(R, o['R'], atol=1e-9, rtol=0), kind
        assert torch.allclose(s, o['s'], rtol=1e-9, atol=0), kind
        assert torch.allclose(t, o['t'], atol=1e-9 * (1 + float(o['t'].abs().max())), rtol=0), kind
    x, y, w = procrustes_problems(2, 300, seed=22, kind='mirror')
    assert bool((torch.linalg.det(O.umeyama64(x, y, w)['M']) < 0).all())


def test_registration_bound_covers_the_wrapper_formula():
    """The wrapper's uncentred-moment formula, evaluated in float64 on the host from exact-ish moments and rounded to fp32, lies
    within registration64's bound (the bound's own consistency, far-from-origin case included)."""
    for kind in ('general', 'planar', 'mirror', 'far', 'half_zero', 'anchor'):
        x, y, w = procrustes_problems(3, 700, seed=23, kind=kind)
        m, dm = O.moments64(x, y, w)
        ref = O.registration64(x, y, w, m, dm)
        R, t, s = _wrapper_formula(m)
        ratios, n = registration_ratios(R, t, s, ref)
        assert n == 3 and max(ratios.values()) <= 1, (kind, ratios)


def _wrapper_formula(m):
    """scene_ops.rigid_registration's arithmetic from the moments, on the host in float64."""
    B = m.shape[0]
    sw = m[:, 0]
    xm, ym = m[:, 1:4] / sw[:, None], m[:, 4:7] / sw[:, None]
    M = m[:, 7:16].reshape(B, 3, 3) - sw[:, None, None] * ym[:, :, None] * xm[:, None, :]
    varx = m[:, 16] - sw * (xm * xm).sum(dim=-1)
    Uu, S, Vh = torch.linalg.svd(M)
    D = torch.ones_like(S)
    D[:, -1] = torch.sign(torch.linalg.det(Uu @ Vh))
    R = Uu @ torch.diag_embed(D) @ Vh
    s = (S * D).sum(dim=-1) / varx
    t = ym - s[:, None] * (R @ xm[:, :, None])[:, :, 0]
    return R.float(), t.float(), s.float()


# ------------------------------------------------------------------------------------------- resolution demonstration
def test_resolution_clean():
    cases = clean_cases()
    # half away from zero, and `<=` in the depth test, on the exact identity scene
    scene, tol, bad = cases['half']
    pts, conf, depth, hw, K, T = flat(scene)
    good = [c.float() for c, _ in O.clean64(pts, conf, depth, hw, K, T, tol, bad)]
    assert O.check_clean(good, pts, conf, depth, hw, K, T, tol, bad)[0] == 0
    for mutant in ('away', 'le'):
        got = [c.float() for c, _ in O.clean64(pts, conf, depth, hw, K, T, tol, bad, mutant=mutant)]
        assert O.check_clean(got, pts, conf, depth, hw, K, T, tol, bad)[0] > 0, mutant
    # parallel semantics on the chain scene
    scene, tol, bad = cases['chain']
    pts, conf, depth, hw, K, T = flat(scene)
    seq = [c.float() for c, _ in O.clean64(pts, conf, depth, hw, K, T, tol, bad)]
    got = [c.float() for c, _ in O.clean64(pts, conf, depth, hw, K, T, tol, bad, parallel=True)]
    assert any(not torch.equal(a, b) for a, b in zip(seq, got))
    assert O.check_clean(got, pts, conf, depth, hw, K, T, tol, bad)[0] > 0
    # image i's width on mixed sizes
    scene, tol, bad = cases['n5_mixed_tol0']
    pts, conf, depth, hw, K, T = flat(scene)
    got = [c.float() for c, _ in O.clean64(pts, conf, depth, hw, K, T, tol, bad, mutant='width')]
    assert O.check_clean(got, pts, conf, depth, hw, K, T, tol, bad)[0] > 0


def test_resolution_procrustes():
    x, y, w = procrustes_problems(5, 2049, seed=24)
    m, dm = O.moments64(x, y, w)
    assert moments_ratio(m, m, dm) == 0
    mut = m.clone()
    mut[2] = O.moments64(x[2:3, :-1], y[2:3, :-1], w[2:3, :-1])[0][0]       # last point of problem 2 dropped
    assert moments_ratio(mut, m, dm) > 1
    wm = torch.cat([w[:1], w[:-1]])                                             # problem b reads problem b - 1's weights
    assert moments_ratio(O.moments64(x, y, wm)[0], m, dm) > 1


def clip_map():
    """A 9 x 9 map, principal point (0, 0), where the 1e-8 clip decides a step.  Every pixel but three is NaN (a zero ray).
    Pixel (1, 0) lies exactly on the ray of focal 128 (x / z = 1 / 128).  Pixels (4, 0) and (8, 8) vote 64 and 256, and since
    |(8, 8)|^2 = 8 |(4, 0)|^2 their votes cancel: every term and sum of step 0 is a small dyadic number, so step 0 returns
    exactly 128.  At f = 128 the first pixel's residual is exactly 0 and its weight is 1 / clip, so step 1 depends on the clip:
    at 1e-8 the two voting pixels move the focal by about 2e-8 of it, at 1e-6 by about 2e-6."""
    pts = torch.full((1, 9, 9, 3), float('nan'))
    pts[0, 0, 1] = torch.tensor([1 / 128, 0.0, 1.0])
    pts[0, 0, 4] = torch.tensor([4 / 64, 0.0, 1.0])
    pts[0, 8, 8] = torch.tensor([8 / 256, 8 / 256, 1.0])
    return pts, torch.zeros((1, 2))


def oracle_chain(pts, pp, W, steps=10, **kw):
    """The fp32-rounded oracle focal after 0..steps steps, each step fed the previous one (kw: a deliberate mistake)."""
    P = pts.reshape(pts.shape[0], -1, 3)
    out = [O.weiszfeld_step64(P, pp, W, **kw)[0].float()]
    for _ in range(steps):
        out.append(O.weiszfeld_step64(P, pp, W, out[-1], **kw)[0].float())
    return out


def test_resolution_weiszfeld():
    pts, pp = weiszfeld_maps(33, 31, seed=25)
    true = oracle_chain(pts, pp, 31)
    assert weiszfeld_chain_ratio(pts, pp, 31, true) <= 1
    # one iteration fewer (`it < steps`): steps = 0 returns the initial 0
    fewer = [torch.zeros(4)] + true[:-1]
    assert weiszfeld_chain_ratio(pts, pp, 31, fewer) > 1
    # NaN rays not zeroed
    assert weiszfeld_chain_ratio(pts, pp, 31, oracle_chain(pts, pp, 31, zero_nonfinite=False)) > 1
    # clip at 1e-6, on the map the GPU test runs for the clip (step 0 is exactly 128 there)
    cp, cpp = clip_map()
    true = oracle_chain(cp, cpp, 9)
    assert float(true[0]) == 128.0 and weiszfeld_chain_ratio(cp, cpp, 9, true) <= 1
    assert weiszfeld_chain_ratio(cp, cpp, 9, oracle_chain(cp, cpp, 9, clip=1e-6)) > 1


def test_resolution_nearest_neighbours():
    pts = nn_points(4097, seed=26)
    q = nn_queries(255, pts, seed=27)
    want = O.nn64(q, pts)
    assert O.check_nn(q, pts, want) == 0
    # highest index on ties: the query on the duplicated point gets 2148 instead of 100
    hi = want.clone()
    dup = (q == pts[100]).all(-1)
    assert bool(dup.any())
    hi[dup] = 2148
    assert O.check_nn(q, pts, hi) > 0
    # the last point of every tile skipped
    skip = pts.clone()
    skip[KTILE - 1::KTILE] = float('nan')
    assert O.check_nn(q, pts, O.nn64(q, skip)) > 0
