"""PnP-RANSAC (dust3r_b200/localization.py, csrc/pnp_core.h), CPU side:

  * the per-thread bodies of the CUDA kernels (csrc/pnp_core.h) are compiled for the HOST (tests/native/pnp_host.cpp, g++
    -ffp-contract=off) and checked over every thread index of small launches against oracle/pnp_float64.py: the sample draws
    exactly, EPnP to 1e-9 on the samples the oracle judges well-conditioned, the inlier counts exactly (points within the
    oracle's undecided band are counted and reported), the stopping rule and the whole loop in rounds of several sizes;
  * the oracle is pinned to OpenCV: its EPnP against cv2.solvePnP(SOLVEPNP_EPNP) on noise-free samples, its inlier rule
    against cv2.projectPoints on float32 points, its loop's result against cv2.solvePnPRansac on the same problems;
  * run_pnp on numpy input equals the reference's run_pnp (restated below), and its <= 4-point and ValueError cases.
The `-m gpu` twin is tests/test_pnp_gpu.py.
"""
import ctypes as C

import cv2
import numpy as np
import pytest

import native_harness
from oracle import pnp_float64 as O

SEED = O.DEFAULT_SEED
P = lambda a: a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope='module')
def host():
    lib = C.CDLL(native_harness.build('pnp_host'))
    d = C.c_double
    lib.pnp_hypotheses_host.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, d, d, d, d, d, C.c_uint64, C.c_int32, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_void_p]
    lib.pnp_epnp_host.argtypes = [C.c_void_p, C.c_void_p, d, d, d, d, C.c_void_p]
    lib.pnp_err2_host.argtypes = [C.c_void_p, d, d, d, d, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.pnp_update_num_iters_host.argtypes = [d, d, C.c_int32, C.c_int32]
    lib.pnp_ransac_host.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, d, d, d, d, d, d, C.c_int32, C.c_uint64, C.c_int32,
                                    C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def _cam(K):
    return float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])


def hypotheses_host(lib, p2, p3, K, thr, h0, m, seed=SEED):
    idx, pose, cnt = np.zeros((m, 5), np.int32), np.zeros((m, 12)), np.zeros(m, np.int32)
    lib.pnp_hypotheses_host(len(p2), P(p2), P(p3), *_cam(K), thr, seed, h0, m, P(idx), P(pose), P(cnt))
    return idx, pose, cnt


def ransac_host(lib, p2, p3, K, thr, max_iters=10_000, round_=1024, conf=0.9999, seed=SEED):
    res, pose, mask = np.zeros(4, np.int32), np.zeros(12), np.zeros(len(p2), np.uint8)
    lib.pnp_ransac_host(len(p2), P(p2), P(p3), *_cam(K), thr, conf, max_iters, seed, round_, P(res), P(pose), P(mask))
    return res, pose, mask.astype(bool)


# (n, inlier ratio, noise px, planar, share of outliers behind the camera)
CASES = [(5, 1.0, 0.0, False, 0.0), (6, 1.0, 1.0, False, 0.0), (40, 0.5, 1.0, False, 0.5), (300, 0.2, 0.0, False, 0.0),
         (500, 0.05, 1.0, False, 0.0), (800, 0.5, 1.0, True, 0.0), (1000, 1.0, 0.0, True, 0.0)]


def compare_hypotheses(idx, pose, cnt, p2, p3, K, thr, h0, seed=SEED):
    """Kernel-side hypotheses against the oracle: (undecided points met, ill-conditioned samples skipped, worst EPnP error)."""
    fx, fy, cx, cy = _cam(K)
    undecided = skipped = 0
    worst = 0.0
    for i in range(len(idx)):
        oi = O.sample_indices(seed, h0 + i, len(p2))
        assert list(idx[i]) == oi, (h0 + i, idx[i], oi)
        ref, good = O.epnp_conditioned(p3[oi].astype(np.float64), p2[oi].astype(np.float64), fx, fy, cx, cy)
        if cnt[i] < 0:   # invalid on the kernel side: the oracle must not call it well-conditioned
            assert not good or ref is None, h0 + i
            continue
        assert np.all(np.isfinite(pose[i]))
        R, t = pose[i, :9].reshape(3, 3), pose[i, 9:]
        assert np.allclose(R @ R.T, np.eye(3), atol=1e-9)
        # the count replayed in float64 from the kernel's pose: equal outside the undecided band
        err = O.reproj_err2(R, t, fx, fy, cx, cy, p3, p2)
        inl = err <= O.thr2_of(thr)
        und = O.undecided(R, t, fx, fy, cx, cy, p3, p2, thr, rel=1e-15)
        undecided += int(und.sum())
        assert abs(int(inl.sum()) - int(cnt[i])) <= int(und.sum()), (h0 + i, inl.sum(), cnt[i])
        if not good:
            skipped += 1
            continue
        a = np.hstack([ref[0].ravel(), ref[1]])
        worst = max(worst, float(np.abs(pose[i] - a).max() / max(1.0, np.abs(a).max())))
    assert worst <= 1e-9, worst
    return undecided, skipped, worst


@pytest.mark.parametrize('case', CASES, ids=[f'n{c[0]}-in{c[1]}-noise{c[2]}-planar{int(c[3])}-behind{c[4]}' for c in CASES])
def test_native_hypotheses_equal_oracle(host, case):
    n, ratio, noise, planar, behind = case
    p2, p3, K, _, _, _ = O.synth_problem(n, ratio, noise, seed=n, planar=planar, behind=behind)
    for h0, m in ((0, 96), (1000, 17)):
        idx, pose, cnt = hypotheses_host(host, p2, p3, K, 5.0, h0, m)
        und, skipped, worst = compare_hypotheses(idx, pose, cnt, p2, p3, K, 5.0, h0)
        print(f'{case} h0={h0}: undecided points {und}, ill-conditioned samples skipped {skipped}/{m}, worst EPnP {worst:.1e}')


def test_native_collinear_sample_is_invalid_never_nan(host):
    rng = np.random.default_rng(0)
    s = rng.uniform(-1, 1, size=50)
    p3 = (np.array([0.3, -0.2, 5.0]) + s[:, None] * np.array([1.0, 0.5, 0.2])).astype(np.float32)
    p2 = (np.array([320.0, 240.0]) + 100 * s[:, None] * np.array([1.0, 0.5])).astype(np.float32)
    K = np.array([[500, 0, 320], [0, 500, 240], [0, 0, 1.0]])
    idx, pose, cnt = hypotheses_host(host, p2, p3, K, 5.0, 0, 64)
    assert np.all(np.isfinite(pose))
    res, bpose, mask = ransac_host(host, p2, p3, K, 5.0, max_iters=300)
    assert np.all(np.isfinite(bpose))
    assert res[0] == -1 or res[1] >= 5


def test_native_identical_points_are_invalid(host):
    p3 = np.tile(np.float32([[0.1, 0.2, 4.0]]), (8, 1))
    p2 = np.tile(np.float32([[300.0, 200.0]]), (8, 1))
    K = np.array([[500, 0, 320], [0, 500, 240], [0, 0, 1.0]])
    idx, pose, cnt = hypotheses_host(host, p2, p3, K, 5.0, 0, 8)
    assert np.all(cnt == -1) and np.all(pose == 0)
    res, bpose, mask = ransac_host(host, p2, p3, K, 5.0, max_iters=20)
    assert list(res) == [-1, 0, 20, 1] and not mask.any()


def test_native_error_equals_oracle_bitwise(host):
    p2, p3, K, R, t, _ = O.synth_problem(4000, 0.5, 2.0, seed=7, behind=0.5)
    p3[:5] = [[0, 0, 0]] * 5      # z = t_z of zero would divide by 0: OpenCV uses 1, checked below with t_z = 0
    for Rt in (np.hstack([R.ravel(), t]), np.hstack([R.ravel(), t[:2], 0.0])):
        err = np.zeros(len(p2), np.float32)
        host.pnp_err2_host(P(np.ascontiguousarray(Rt)), *_cam(K), len(p2), P(p2), P(p3), P(err))
        ref = O.reproj_err2(Rt[:9].reshape(3, 3), Rt[9:], *_cam(K), p3, p2)
        np.testing.assert_array_equal(err.view(np.int32), ref.view(np.int32))


def test_oracle_inlier_rule_equals_cv2_projectpoints():
    p2, p3, K, R, t, _ = O.synth_problem(5000, 0.5, 2.0, seed=8)
    rvec = cv2.Rodrigues(R)[0]
    R2 = cv2.Rodrigues(rvec)[0]       # the callback's model is (rvec, tvec): project with the round-tripped R
    proj = cv2.projectPoints(p3, rvec, t, K, None)[0].reshape(-1, 2)
    assert proj.dtype == np.float32
    du, dv = p2[:, 0] - proj[:, 0], p2[:, 1] - proj[:, 1]
    err_cv = du * du + dv * dv
    err = O.reproj_err2(R2, t, *_cam(K), p3, p2)
    np.testing.assert_array_equal(err, err_cv)
    thr = 3.0
    assert np.array_equal(err <= O.thr2_of(thr), err_cv <= np.float32(thr * thr))


def test_oracle_epnp_equals_cv2_noise_free():
    rng = np.random.default_rng(3)
    worst = 0.0
    for trial in range(40):
        p2, p3, K, R, t, _ = O.synth_problem(100, 1.0, 0.0, seed=trial)
        idx = rng.choice(100, 5, replace=False)
        pw = p3[idx].astype(np.float64)
        Xc = pw @ R.T + t
        uv = np.stack([K[0, 0] * Xc[:, 0] / Xc[:, 2] + K[0, 2], K[1, 1] * Xc[:, 1] / Xc[:, 2] + K[1, 2]], 1)
        R_o, t_o = O.epnp(pw, uv, *_cam(K))
        ok, rvec, tvec = cv2.solvePnP(pw, uv, K, None, flags=cv2.SOLVEPNP_EPNP)
        assert ok
        a, b = np.hstack([R_o.ravel(), t_o]), np.hstack([cv2.Rodrigues(rvec)[0].ravel(), tvec.ravel()])
        worst = max(worst, np.abs(a - b).max() / np.abs(b).max())
    assert worst <= 1e-6, worst


def test_native_epnp_noise_free_equals_truth(host):
    for trial in range(20):
        p2, p3, K, R, t, _ = O.synth_problem(50, 1.0, 0.0, seed=100 + trial, planar=trial % 2 == 1)
        pw = np.ascontiguousarray(p3[:5].astype(np.float64))
        Xc = pw @ R.T + t
        uv = np.ascontiguousarray(np.stack([K[0, 0] * Xc[:, 0] / Xc[:, 2] + K[0, 2], K[1, 1] * Xc[:, 1] / Xc[:, 2] + K[1, 2]], 1))
        Rt = np.zeros(12)
        assert host.pnp_epnp_host(P(pw), P(uv), *_cam(K), P(Rt)) == 1
        truth = np.hstack([R.ravel(), t])
        assert np.abs(Rt - truth).max() <= 1e-6 * max(1, np.abs(truth).max()), (trial, np.abs(Rt - truth).max())


def test_native_update_num_iters_equals_oracle(host):
    for conf in (0.5, 0.99, 0.9999, 1 - 1e-12):
        for ep in (0.0, 1e-9, 0.05, 0.3, 0.5, 0.8, 0.95, 0.999, 1.0):
            for it in (1, 10, 10_000):
                assert host.pnp_update_num_iters_host(conf, ep, 5, it) == O.update_num_iters(conf, ep, 5, it), (conf, ep, it)


@pytest.mark.parametrize('ratio', [1.0, 0.5, 0.2])
def test_native_loop_equals_oracle_loop_in_any_round_size(host, ratio):
    p2, p3, K, _, _, _ = O.synth_problem(400, ratio, 1.0, seed=11)
    fx, fy, cx, cy = _cam(K)
    results = {r: ransac_host(host, p2, p3, K, 5.0, max_iters=3000, round_=r) for r in (1, 7, 64, 1024)}
    res, pose, mask = results[1024]
    for r, (res_r, pose_r, mask_r) in results.items():
        assert list(res_r) == list(res) and np.array_equal(pose_r, pose) and np.array_equal(mask_r, mask), r
    # the sequential loop over the same hypotheses (their counts from the harness), and over the oracle's own counts
    _, _, cnt = hypotheses_host(host, p2, p3, K, 5.0, 0, int(res[2]))
    assert O.ransac_loop(lambda h: int(cnt[h]), len(p2), 0.9999, 3000) == (res[0], res[1], res[2])
    if res[2] <= 400:
        best, count, evaluated, opose, omask = O.ransac(p2, p3, fx, fy, cx, cy, 5.0, max_iters=3000)
        assert (best, count, evaluated) == tuple(res[:3])
        assert np.array_equal(omask, mask)
    assert res[3] == 1 and mask.sum() == res[1]


def test_native_iteration_cap_and_early_stop(host):
    p2, p3, K, _, _, _ = O.synth_problem(500, 0.1, 0.5, seed=12)
    for cap in (1, 5, 33, 100):
        res, _, _ = ransac_host(host, p2, p3, K, 5.0, max_iters=cap, round_=16)
        assert res[2] == cap
    p2, p3, K, _, _, _ = O.synth_problem(500, 1.0, 0.0, seed=13)
    res, _, mask = ransac_host(host, p2, p3, K, 5.0, max_iters=10_000)
    assert res[0] == 0 and res[1] == 500 and res[2] == 1 and mask.all()   # every point an inlier: niters drops to 0


def test_native_loop_agrees_with_cv2(host):
    for ratio, noise, seed in ((0.95, 0.5, 1), (0.5, 1.0, 2), (0.3, 0.5, 3)):
        p2, p3, K, R, t, _ = O.synth_problem(2000, ratio, noise, seed=seed)
        res, pose, mask = ransac_host(host, p2, p3, K, 5.0)
        ok, rvec, tvec, inl = cv2.solvePnPRansac(p3, p2, K, None, flags=cv2.SOLVEPNP_SQPNP, iterationsCount=10_000,
                                                 reprojectionError=5.0, confidence=0.9999)
        assert ok and res[0] >= 0
        assert abs(int(mask.sum()) - len(inl)) <= 0.01 * len(inl), (mask.sum(), len(inl))


# ---- run_pnp on numpy input ----

def reference_run_pnp(pts2D, pts3D, K, distortion=None, reprojectionError=5):
    """dust3r_visloc/localization.py:30-52, mode 'cv2', restated."""
    try:
        if len(pts2D) > 4:
            if distortion is not None:
                pts2D = cv2.undistortPoints(np.copy(pts2D), K, np.array(distortion), R=None, P=K).reshape((-1, 2))
            success, r_pose, t_pose, _ = cv2.solvePnPRansac(pts3D, pts2D, K, None, flags=cv2.SOLVEPNP_SQPNP,
                                                            iterationsCount=10_000, reprojectionError=reprojectionError,
                                                            confidence=0.9999)
            if not success:
                return False, None
            r_pose = cv2.Rodrigues(r_pose)[0]
            RT = np.r_[np.c_[r_pose, t_pose], [(0, 0, 0, 1)]]
            return True, np.linalg.inv(RT)
        return False, None
    except Exception:
        return False, None


@pytest.mark.parametrize('distortion', [None, [0.01, -0.005, 0.001, 0.0005]])
def test_run_pnp_numpy_equals_reference(distortion):
    from dust3r_b200.localization import run_pnp
    p2, p3, K, _, _, _ = O.synth_problem(3000, 0.5, 1.0, seed=21)
    for thr in (5, 2.5):
        ok_a, a = run_pnp(p2, p3, K, distortion, 'cv2', thr)
        ok_b, b = reference_run_pnp(p2, p3, K, distortion, thr)
        assert ok_a == ok_b and np.array_equal(a, b)


def test_run_pnp_small_and_invalid_input():
    from dust3r_b200.localization import run_pnp
    p2, p3, K, _, _, _ = O.synth_problem(50, 1.0, 0.0, seed=22)
    assert run_pnp(p2[:4], p3[:4], K) == (False, None)
    assert run_pnp(p2[:0], p3[:0], K) == (False, None)
    for bad in ('2d', '3d', 'K'):
        q2, q3, KK = p2.copy(), p3.copy(), K.copy()
        {'2d': q2, '3d': q3, 'K': KK}[bad][0, 0] = np.nan
        with pytest.raises(ValueError):
            run_pnp(q2, q3, KK)
    with pytest.raises(ValueError):
        run_pnp(p2, p3, K, mode='poselib')


def test_aggregate_stats_and_pose_error():
    from dust3r_b200.localization import aggregate_stats, get_pose_error
    rng = np.random.default_rng(0)
    for _ in range(20):
        A = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        A *= np.linalg.det(A)
        B = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        B *= np.linalg.det(B)
        Ta, Tb = np.eye(4), np.eye(4)
        Ta[:3, :3], Tb[:3, :3] = A, B
        Ta[:3, 3], Tb[:3, 3] = rng.normal(size=3), rng.normal(size=3)
        te, ae = get_pose_error(Ta, Tb)
        ang = np.degrees(np.arccos(np.clip((np.trace(A.T @ B) - 1) / 2, -1, 1)))
        assert abs(float(te) - np.linalg.norm(Ta[:3, 3] - Tb[:3, 3])) <= 1e-12
        assert abs(float(ae) - ang) <= 1e-6
    s = aggregate_stats('x', [0.05, 0.2, 1.0, float('inf')], [0.5, 1.5, 4.0, float('inf')])
    assert 'acc@0.1m,1deg=25.000' in s and 'acc@0.25m,2deg=50.000' in s and 'acc@5m,10deg=75.000' in s
