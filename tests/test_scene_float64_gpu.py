"""The four scene kernels of csrc/scene_ops.cu element by element against the float64 oracle (oracle/scene_float64.py), called
through ctypes with buffers the test allocates: every output buffer has a guard region after it that must keep its byte pattern,
and every input must be unchanged after the call.

  d3r_procrustes_moments  every one of the 17 moments within its bound, at P = 1, 2, 255, the chunk edges 2047 / 2048 / 2049
                          (bx = ceil(P / 2048) CTAs per problem), 131072 / 131073 (64 CTAs, then the grid-stride loop) and
                          196608, B = 1 and 5 problems that each have their own rotation, scale, translation and weights, planar,
                          mirrored (D = -1), far-from-origin and half-zero-weight clouds, and the anchor-registration shape
                          (P = 2n, no weights); R, t, s of rigid_points_registration within their bounds; 65535 problems run and
                          65536 raise.  The moments are atomicAdd'ed across CTAs, so reruns need not be bit-identical.
  d3r_weiszfeld_focal     steps = k for k = 0..10, each against one oracle step fed the device's steps = k - 1 result (sound
                          because the reduction order is fixed: two runs are asserted bit-identical first), at 1x1, 5x7, 32x32
                          (one CTA of 1024 threads), 33x31, 384x512 and 512x384, four maps with different focals and off-centre
                          principal points, with 0/0, x/0, NaN and zero-ray pixels; a map whose step 0 is exactly 128 and
                          where one pixel's residual at 128 is exactly 0, so that step 1 depends on the 1e-8 residual clip;
                          estimate_focal_knowing_depth end to end with its focal clip; steps < 0 raises.
  d3r_clean_pointcloud    every decided pixel bit-equal to the oracle (image i against the device's own final confidences of
                          images < i), every undecided pixel holding one of its two possible values; n = 1, mixed sizes whose
                          areas are not multiples of 256, points behind cameras, off the images, NaN points and depths,
                          tol 0 / 0.001 / 0.3, bad_conf 0 / 1.5, exact half-integer projections, and a chain scene on which the
                          sequential oracle equals the kernel exactly and differs from parallel semantics; tol = 1 and tol < 0
                          raise.
  d3r_nearest_neighbours  every query's index within eps of the float64 minimum, the lowest index among exact duplicates (100 and
                          2148 straddle the first tile), all-identical points, queries on points (distance 0), NaN rows, M and N
                          around the 2048-point tile and the 256-thread CTA, and one 196608 x 196608 call sampled against a
                          float64 k-d tree; find_reciprocal_matches equals the oracle's reciprocity wherever no near-tie is
                          involved.

Every bound constant is derived in oracle/scene_float64.py; none is fitted.  Worst err / bound observed on an H100 80GB HBM3
(700 W), over the whole file (printed at the end of the module):
    Procrustes moments 0.043   R 0.952   t 0.952   s 0.871  (R, t and s are dominated by the final fp32 rounding, whose
                       bound u |x| is reached up to a factor ~1 just above a power of two)
    Weiszfeld focal    0.184
    clean_pointcloud   at most 1 undecided pixel per case: 1 in each of two cases (n5_mixed_tol0: 1 of 3299 cut pixels;
                       n5_mixed_tol0.3_bad1.5: 1 of 26), 0 in the others; every decided pixel matched exactly."""
from collections import defaultdict

import numpy as np
import pytest
import torch

from dust3r_b200 import _lib
from oracle import scene_float64 as O

from test_scene_float64_host import (clean_cases, clip_map, flat, moments_ratio, nn_points, nn_queries, procrustes_problems,
                                     registration_ratios, weiszfeld_chain_ratio, weiszfeld_maps)

pytestmark = pytest.mark.gpu

GUARD = 4096
WORST = defaultdict(float)


@pytest.fixture(scope='module', autouse=True)
def report_worst():
    yield
    print('\nworst err / bound (and largest undecided count):')
    for k, v in sorted(WORST.items()):
        print(f'  {k:28s} {v:.3g}')


def _bits(t):
    return t.contiguous().view(torch.uint8).clone()


class Out:
    """An output buffer of n elements followed by GUARD bytes of 0xA5; `init` fills the first part."""

    def __init__(self, n, dtype, dev, init=None):
        self.n, self.dtype = n, dtype
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        self.raw = torch.full((nbytes + GUARD,), 0xA5, dtype=torch.uint8, device=dev)
        self.t = self.raw[:nbytes].view(dtype)
        if init is not None:
            self.t.copy_(init.reshape(-1))

    def ptr(self):
        return self.t.data_ptr()

    def done(self):
        torch.cuda.synchronize()
        assert bool((self.raw[self.t.numel() * self.t.element_size():] == 0xA5).all()), 'write past the output buffer'
        return self.t.cpu()


def call(name, ins, out, *args, dev):
    """launch(name, *args) and check the guard of `out` and that every tensor of `ins` is unchanged."""
    before = [_bits(t) for t in ins]
    _lib.launch(dev, name, *args)
    res = out.done()
    for t, b in zip(ins, before):
        assert torch.equal(_bits(t), b), 'input modified'
    return res


# ------------------------------------------------------------------------------------------------------------ Procrustes
def moments_call(x, y, w, dev):
    B, P = w.shape
    xd, yd, wd = (t.to(dev).contiguous() for t in (x, y, w))
    out = Out(17 * B, torch.float64, dev)
    return call('d3r_procrustes_moments', [xd, yd, wd], out, B, P, xd.data_ptr(), yd.data_ptr(), wd.data_ptr(), out.ptr(),
                dev=dev).reshape(B, 17)


def check_procrustes(x, y, w, dev, weights=True):
    from dust3r_b200.cloud_opt.commons import rigid_points_registration
    m, dm = O.moments64(x, y, w)
    got = moments_call(x, y, w, dev)
    r = moments_ratio(got, m, dm)
    WORST['procrustes moments'] = max(WORST['procrustes moments'], r)
    assert r <= 1, r
    if x.shape[1] < 3:
        return 0
    kw = dict(weights=w.to(dev)) if weights else {}
    R, t, s = rigid_points_registration(x.to(dev), y.to(dev), compute_scaling=True, **kw)
    ref = O.registration64(x, y, w, m, dm)
    ratios, n = registration_ratios(R.cpu(), t.cpu(), s.cpu(), ref)
    for k, v in ratios.items():
        WORST[f'procrustes {k}'] = max(WORST[f'procrustes {k}'], v)
        assert v <= 1, (k, v)
    return n


@pytest.mark.parametrize('P', [1, 2, 255, 2047, 2048, 2049, 131072, 131073, 196608])
@pytest.mark.parametrize('B', [1, 5])
def test_procrustes_sizes(P, B, cuda_device):
    x, y, w = procrustes_problems(B, P, seed=P + B)
    n = check_procrustes(x, y, w, cuda_device)
    if P >= 255:
        assert n == B                        # every problem's R, t, s was checked


@pytest.mark.parametrize('kind', ['planar', 'mirror', 'far', 'half_zero'])
@pytest.mark.parametrize('P', [2049, 131073])
def test_procrustes_geometry(kind, P, cuda_device):
    x, y, w = procrustes_problems(5, P, seed=P + 7, kind=kind)
    assert check_procrustes(x, y, w, cuda_device) == 5


def test_procrustes_anchor_registration(cuda_device):
    """init_im_poses' anchor registration: P = 2n camera centres and offsets, no weights."""
    x, y, w = procrustes_problems(1, 16, seed=31, kind='anchor')
    assert check_procrustes(x, y, w, cuda_device, weights=False) == 1


def test_procrustes_problem_limit(cuda_device):
    B = 65535
    g = torch.Generator().manual_seed(33)
    xb, yb = torch.randn((B, 1, 3), generator=g), torch.randn((B, 1, 3), generator=g)
    wb = torch.rand((B, 1), generator=g)
    m, dm = O.moments64(xb, yb, wb)
    assert moments_ratio(moments_call(xb, yb, wb, cuda_device), m, dm) <= 1
    xb, yb, wb = (torch.cat([t, t[:1]]) for t in (xb, yb, wb))
    with pytest.raises(_lib.D3RError, match='too many problems'):
        moments_call(xb, yb, wb, cuda_device)


# -------------------------------------------------------------------------------------------------------------- Weiszfeld
def focal_call(pts, pp, steps, dev):
    B, H, W, _ = pts.shape
    pd, cd = pts.to(dev).contiguous(), pp.to(dev).contiguous()
    out = Out(B, torch.float32, dev)
    return call('d3r_weiszfeld_focal', [pd, cd], out, B, H, W, pd.data_ptr(), cd.data_ptr(), steps, out.ptr(), dev=dev)


@pytest.mark.parametrize('shape', [(1, 1), (5, 7), (32, 32), (33, 31), (384, 512), (512, 384)])
def test_weiszfeld_every_step(shape, cuda_device):
    H, W = shape
    pts, pp = weiszfeld_maps(H, W, seed=40 + H * W)
    a, b = focal_call(pts, pp, 10, cuda_device), focal_call(pts, pp, 10, cuda_device)
    assert torch.equal(_bits(a), _bits(b)), 'reduction order not fixed'
    chain = [focal_call(pts, pp, k, cuda_device) for k in range(11)]
    assert torch.equal(_bits(chain[-1]), _bits(a))
    r = weiszfeld_chain_ratio(pts, pp, W, chain)
    WORST['weiszfeld focal'] = max(WORST['weiszfeld focal'], r)
    assert r <= 1, r


def test_weiszfeld_residual_clip(cuda_device):
    """A map on which step 0 is exactly 128 and one pixel's residual at 128 is exactly 0: step 1 weights that pixel 1 / 1e-8f,
    and a different clip moves the focal far beyond its bound (tests/test_scene_float64_host.py: clip_map)."""
    pts, pp = clip_map()
    a, b = focal_call(pts, pp, 10, cuda_device), focal_call(pts, pp, 10, cuda_device)
    assert torch.equal(_bits(a), _bits(b)), 'reduction order not fixed'
    chain = [focal_call(pts, pp, k, cuda_device) for k in range(11)]
    assert float(chain[0]) == 128.0
    r = weiszfeld_chain_ratio(pts, pp, 9, chain)
    WORST['weiszfeld focal'] = max(WORST['weiszfeld focal'], r)
    assert r <= 1, r


def test_weiszfeld_end_to_end_with_clip(cuda_device):
    import math
    from dust3r_b200.post_process import estimate_focal_knowing_depth
    H, W = 33, 31
    pts, pp = weiszfeld_maps(H, W, seed=40 + H * W)
    f10 = focal_call(pts, pp, 10, cuda_device)
    fov60 = max(H, W) / (2 * math.tan(math.radians(60) / 2))
    lo, hi = float(f10.min()) * 1.01 / fov60, float(f10.max()) * 0.99 / fov60
    got = estimate_focal_knowing_depth(pts.to(cuda_device), pp.to(cuda_device), focal_mode='weiszfeld', min_focal=lo,
                                       max_focal=hi).cpu()
    want = f10.clip(min=lo * fov60, max=hi * fov60)
    assert torch.equal(got, want) and not torch.equal(want, f10)


def test_weiszfeld_negative_steps_raise(cuda_device):
    pts, pp = weiszfeld_maps(5, 7, seed=41)
    with pytest.raises(_lib.D3RError, match='bad arguments'):
        focal_call(pts, pp, -1, cuda_device)


# ------------------------------------------------------------------------------------------------------- clean_pointcloud
def clean_call(scene, tol, bad, dev):
    pts, conf, depth, hw, K, T = flat(scene)
    n = len(pts)
    areas = [h * w for h, w in hw]
    off = torch.tensor(np.concatenate([[0], np.cumsum(areas)]), dtype=torch.int64, device=dev)
    hwd = torch.tensor(hw, dtype=torch.int32, device=dev)
    pd = torch.cat(pts).to(dev).contiguous()
    dd = torch.cat(depth).to(dev).contiguous()
    Kd, Td = K.reshape(n, 9).to(dev).contiguous(), T.reshape(n, 16).to(dev).contiguous()
    out = Out(sum(areas), torch.float32, dev, init=torch.cat(conf).to(dev))
    res = call('d3r_clean_pointcloud', [off, hwd, pd, dd, Kd, Td], out, n, hwd.data_ptr(), off.data_ptr(), max(areas),
               pd.data_ptr(), out.ptr(), dd.data_ptr(), Kd.data_ptr(), Td.data_ptr(), float(tol), float(bad), dev=dev)
    return [res[a:b] for a, b in zip(off[:-1].tolist(), off[1:].tolist())]


@pytest.mark.parametrize('name', list(clean_cases()))
def test_clean_pointcloud(name, cuda_device):
    scene, tol, bad = clean_cases()[name]
    got = clean_call(scene, tol, bad, cuda_device)
    pts, conf, depth, hw, K, T = flat(scene)
    wrong, und, bad_und, cut = O.check_clean(got, pts, conf, depth, hw, K, T, tol, bad)
    print(f'{name}: {und} undecided pixels, {cut} cut')
    WORST['clean undecided pixels'] = max(WORST['clean undecided pixels'], und)
    assert wrong == 0 and bad_und == 0, (wrong, bad_und)
    assert und <= max(2, cut // 50), (und, cut)
    if name == 'n1':
        assert torch.equal(got[0], conf[0])
    else:
        assert cut > 0
    if name in ('half', 'chain'):
        seq = O.clean64(pts, conf, depth, hw, K, T, tol, bad)
        assert all(not u.any() and torch.equal(g, c.float()) for g, (c, u) in zip(got, seq))
    if name == 'chain':
        par = O.clean64(pts, conf, depth, hw, K, T, tol, bad, parallel=True)
        assert any(not torch.equal(g, c.float()) for g, (c, _) in zip(got, par))


def test_clean_pointcloud_tol_range(cuda_device):
    scene = clean_cases()['chain'][0]
    for tol in (1.0, -0.001):
        with pytest.raises(_lib.D3RError, match='tol'):
            clean_call(scene, tol, 0.0, cuda_device)


# --------------------------------------------------------------------------------------------------- nearest neighbours
def nn_call(q, p, dev):
    qd, pd = q.to(dev).contiguous(), p.to(dev).contiguous()
    out = Out(q.shape[0], torch.int32, dev)
    return call('d3r_nearest_neighbours', [qd, pd], out, q.shape[0], p.shape[0], qd.data_ptr(), pd.data_ptr(), out.ptr(),
                dev=dev)


@pytest.mark.parametrize('M', [1, 2047, 2048, 2049, 4097, 5000])
@pytest.mark.parametrize('N', [1, 255, 257, 5000])
def test_nearest_neighbours_shapes(N, M, cuda_device):
    p = nn_points(M, seed=M)
    q = nn_queries(N, p, seed=N + M)
    got = nn_call(q, p, cuda_device)
    assert O.check_nn(q, p, got) == 0
    if M > 2148 and N > 1:
        on_dup = (q == p[100]).all(-1)
        assert bool(on_dup.any()) and bool((got[on_dup] == 100).all())
    on_pt = (q[:, None, :] == p[None, :, :]).all(-1).any(-1)
    k = got.long()[on_pt]
    assert bool(((q[on_pt] - p[k]) == 0).all())


def test_nearest_neighbours_edges(cuda_device):
    # all points identical
    p = torch.full((4097, 3), 0.5)
    q = torch.randn((300, 3), generator=torch.Generator().manual_seed(50))
    assert bool((nn_call(q, p, cuda_device) == 0).all())
    # NaN rows: never chosen; a NaN query, or all points NaN, gets 0
    p = nn_points(2049, seed=51)
    p[[0, 7, 2047, 2048]] = float('nan')
    q = nn_queries(257, p, seed=52)
    q[[3, 100]] = float('nan')
    got = nn_call(q, p, cuda_device)
    assert O.check_nn(q, p, got) == 0
    assert int(got[3]) == 0 and int(got[100]) == 0 and not bool(torch.isin(got, torch.tensor([7, 2047, 2048], dtype=torch.int32)).any())
    assert bool((nn_call(q, torch.full((300, 3), float('nan')), cuda_device) == 0).all())


@pytest.mark.timeout(1200)
def test_nearest_neighbours_full_map(cuda_device):
    """One 196608 x 196608 call (a 512x384 map against another), sampled on 4096 queries against a float64 k-d tree."""
    from scipy.spatial import cKDTree
    g = torch.Generator().manual_seed(53)
    p = torch.randn((196608, 3), generator=g)
    q = p + 0.01 * torch.randn((196608, 3), generator=g)
    got = nn_call(q, p, cuda_device)
    idx = torch.randperm(196608, generator=g)[:4096]
    d, _ = cKDTree(p.double().numpy()).query(q[idx].double().numpy(), k=2)
    assert O.check_nn(q, p, got, idx=idx, d12=torch.from_numpy(d)) == 0


def test_reciprocal_matches_equal_oracle(cuda_device):
    from dust3r_b200.utils.geometry import find_reciprocal_matches
    g = torch.Generator().manual_seed(54)
    P1 = torch.randn((5000, 3), generator=g)
    P2 = torch.cat((P1[:3000] + 0.01 * torch.randn((3000, 3), generator=g), torch.randn((1500, 3), generator=g)))
    P1[2148] = P1[100]
    m, nn, cnt = find_reciprocal_matches(P1.to(cuda_device), P2.to(cuda_device))
    nn1, nn2 = O.nn64(P1, P2), O.nn64(P2, P1)
    tie1, tie2 = O.near_tie(P1, P2), O.near_tie(P2, P1)
    want = nn1[nn2] == torch.arange(len(P2))
    clear = ~tie2 & ~tie1[nn2]
    assert int(clear.sum()) > 4000
    assert torch.equal(nn.cpu()[~tie2], nn2[~tie2])
    assert torch.equal(m.cpu()[clear], want[clear])
    assert cnt == int(m.sum())
