"""PnP-RANSAC kernels on the GPU (csrc/pnp_ops.cu, dust3r_b200.localization.pnp_ransac / run_pnp):

  * d3r_pnp_hypotheses against oracle/pnp_float64.py over N = 5 .. 100 000, inlier ratios 1 / 0.5 / 0.2 / 0.05, noise 0 and
    1 px, planar scenes, outliers behind the camera: sample indices exactly, counts exactly outside the undecided band
    (reported), EPnP to 1e-9 on the samples the oracle judges well-conditioned (the skipped ones reported);
  * d3r_pnp_ransac against the sequential loop of the oracle over the same hypotheses: best index, count, evaluated count;
  * run_pnp on CUDA tensors against cv2.solvePnPRansac: both succeed, pose within 0.1 deg / 1 % of scene scale of the ground
    truth, inlier counts within 1 %; its pose is cv2.solvePnP(SQPNP) on the returned inliers bit for bit; repeat calls give
    the same bits; iteration cap, early stop and a degenerate input.
"""
import cv2
import numpy as np
import pytest
import torch

from oracle import pnp_float64 as O
from test_pnp_host import CASES, compare_hypotheses

pytestmark = pytest.mark.gpu
SEED = O.DEFAULT_SEED


def _hypotheses(dev, p2, p3, K, thr, h0, m, seed=SEED):
    from dust3r_b200 import _lib
    t2, t3 = torch.from_numpy(p2).to(dev), torch.from_numpy(p3).to(dev)
    idx = torch.empty((m, 5), dtype=torch.int32, device=dev)
    pose = torch.empty((m, 12), dtype=torch.float64, device=dev)
    cnt = torch.empty((m,), dtype=torch.int32, device=dev)
    _lib.launch(dev, 'd3r_pnp_hypotheses', len(p2), t2.data_ptr(), t3.data_ptr(), float(K[0, 0]), float(K[1, 1]), float(K[0, 2]),
                float(K[1, 2]), float(thr), int(seed), int(h0), int(m), idx.data_ptr(), pose.data_ptr(), cnt.data_ptr())
    return idx.cpu().numpy(), pose.cpu().numpy(), cnt.cpu().numpy()


GPU_CASES = CASES + [(100_000, 0.5, 1.0, False, 0.0), (100_000, 0.2, 0.0, False, 0.5), (20_000, 0.05, 1.0, True, 0.0)]


@pytest.mark.parametrize('case', GPU_CASES, ids=[f'n{c[0]}-in{c[1]}-noise{c[2]}-planar{int(c[3])}-behind{c[4]}' for c in GPU_CASES])
def test_hypotheses_equal_oracle(cuda_device, case):
    n, ratio, noise, planar, behind = case
    p2, p3, K, _, _, _ = O.synth_problem(n, ratio, noise, seed=n, planar=planar, behind=behind)
    for h0, m in ((0, 96), (4000, 33)):
        idx, pose, cnt = _hypotheses(cuda_device, p2, p3, K, 5.0, h0, m)
        und, skipped, worst = compare_hypotheses(idx, pose, cnt, p2, p3, K, 5.0, h0)
        print(f'{case} h0={h0}: undecided points {und}, ill-conditioned samples skipped {skipped}/{m}, worst EPnP {worst:.1e}')


@pytest.mark.parametrize('ratio,noise', [(1.0, 0.0), (0.5, 1.0), (0.2, 1.0), (0.05, 0.5)])
def test_loop_equals_sequential_loop(cuda_device, ratio, noise):
    from dust3r_b200.localization import pnp_ransac
    n = 20_000
    p2, p3, K, _, _, _ = O.synth_problem(n, ratio, noise, seed=31)
    result, pose, mask = pnp_ransac(torch.from_numpy(p2).to(cuda_device), torch.from_numpy(p3).to(cuda_device), K, 5.0)
    res = result.cpu().numpy()
    _, hp, cnt = _hypotheses(cuda_device, p2, p3, K, 5.0, 0, int(res[2]))
    assert O.ransac_loop(lambda h: int(cnt[h]), n, 0.9999, 10_000) == tuple(int(x) for x in res[:3])
    assert res[3] == 1
    if res[0] >= 0:
        assert np.array_equal(pose.cpu().numpy().reshape(3, 4), np.c_[hp[res[0], :9].reshape(3, 3), hp[res[0], 9:]])
        assert int(mask.sum()) == res[1]
        R, t = hp[res[0], :9].reshape(3, 3), hp[res[0], 9:]
        ref = O.reproj_err2(R, t, K[0, 0], K[1, 1], K[0, 2], K[1, 2], p3, p2) <= O.thr2_of(5.0)
        assert np.array_equal(mask.cpu().numpy(), ref)
    print(f'ratio {ratio}: best {res[0]}, inliers {res[1]}, hypotheses evaluated {res[2]}')


def _rot_err_deg(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1)))


@pytest.mark.parametrize('ratio', [0.95, 0.5, 0.2])
def test_run_pnp_against_cv2(cuda_device, ratio):
    from dust3r_b200.localization import pnp_ransac, run_pnp
    # At 20 % inliers a 5-point sample is clean with probability 0.2^5, so 10 000 hypotheses draw none with probability
    # e^-3.2 ~ 4 %, whatever the generator.  Seed 2 is such a problem for our draws (its best hypothesis has 362 inliers);
    # seeds 1 and 3 draw clean samples.
    for seed in (1, 3):
        p2, p3, K, R, t, _ = O.synth_problem(30_000, ratio, 0.5, seed=seed)
        ok_g, T_g = run_pnp(torch.from_numpy(p2).to(cuda_device), torch.from_numpy(p3).to(cuda_device), K, None, 'cv2', 5)
        ok_c, rvec, tvec, inl = cv2.solvePnPRansac(p3, p2, K, None, flags=cv2.SOLVEPNP_SQPNP, iterationsCount=10_000,
                                                   reprojectionError=5, confidence=0.9999)
        assert ok_g and ok_c
        W = np.linalg.inv(T_g)           # world -> camera
        scale = np.linalg.norm(p3 - p3.mean(0), axis=1).mean()
        assert _rot_err_deg(W[:3, :3], R) <= 0.1 and np.linalg.norm(W[:3, 3] - t) <= 0.01 * scale
        result, _, mask = pnp_ransac(torch.from_numpy(p2).to(cuda_device), torch.from_numpy(p3).to(cuda_device), K, 5)
        assert abs(int(mask.sum()) - len(inl)) <= 0.01 * len(inl), (int(mask.sum()), len(inl))
        # the pose is cv2.solvePnP(SQPNP) on the returned inliers, bit for bit
        keep = mask.cpu().numpy()
        _, rv, tv = cv2.solvePnP(p3[keep].astype(np.float64), p2[keep].astype(np.float64), K, None, flags=cv2.SOLVEPNP_SQPNP)
        ref = np.linalg.inv(np.r_[np.c_[cv2.Rodrigues(rv)[0], tv], [(0, 0, 0, 1)]])
        assert np.array_equal(T_g, ref)
        print(f'ratio {ratio} seed {seed}: inliers {int(mask.sum())} (cv2 {len(inl)}), hypotheses {int(result[2])}')


def test_repeat_calls_same_bits(cuda_device):
    from dust3r_b200.localization import pnp_ransac, run_pnp
    p2, p3, K, _, _, _ = O.synth_problem(50_000, 0.3, 1.0, seed=5)
    t2, t3 = torch.from_numpy(p2).to(cuda_device), torch.from_numpy(p3).to(cuda_device)
    a, b = pnp_ransac(t2, t3, K), pnp_ransac(t2, t3, K)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    ra, rb = run_pnp(t2, t3, K), run_pnp(t2, t3, K)
    assert ra[0] and np.array_equal(ra[1], rb[1])


def test_iteration_cap_and_early_stop(cuda_device):
    from dust3r_b200.localization import pnp_ransac
    p2, p3, K, _, _, _ = O.synth_problem(5000, 0.05, 0.5, seed=6)
    t2, t3 = torch.from_numpy(p2).to(cuda_device), torch.from_numpy(p3).to(cuda_device)
    for cap in (1, 7, 1024, 1025, 3000):
        result, _, _ = pnp_ransac(t2, t3, K, max_iters=cap)
        assert int(result[2]) == cap and int(result[3]) == 1
    p2, p3, K, _, _, _ = O.synth_problem(5000, 1.0, 0.0, seed=7)
    result, _, mask = pnp_ransac(torch.from_numpy(p2).to(cuda_device), torch.from_numpy(p3).to(cuda_device), K)
    assert result.tolist() == [0, 5000, 1, 1] and bool(mask.all())
    p2, p3, K, _, _, _ = O.synth_problem(5, 1.0, 0.0, seed=8)   # 5 points: one EPnP on all of them, every point an inlier
    result, _, mask = pnp_ransac(torch.from_numpy(p2).to(cuda_device), torch.from_numpy(p3).to(cuda_device), K)
    assert result.tolist() == [0, 5, 1, 1] and bool(mask.all())


def test_degenerate_input_fails_or_is_finite(cuda_device):
    from dust3r_b200.localization import pnp_ransac, run_pnp
    rng = np.random.default_rng(0)
    s = rng.uniform(-1, 1, size=2000)
    p3 = (np.array([0.3, -0.2, 5.0]) + s[:, None] * np.array([1.0, 0.5, 0.2])).astype(np.float32)
    p2 = (np.array([320.0, 240.0]) + 100 * s[:, None] * np.array([1.0, 0.5])).astype(np.float32)
    K = np.array([[500, 0, 320], [0, 500, 240], [0, 0, 1.0]])
    t2, t3 = torch.from_numpy(p2).to(cuda_device), torch.from_numpy(p3).to(cuda_device)
    result, pose, _ = pnp_ransac(t2, t3, K, max_iters=2000)
    assert bool(torch.isfinite(pose).all())
    ok, T = run_pnp(t2, t3, K)
    assert (not ok and T is None) or np.all(np.isfinite(T))
    with pytest.raises(ValueError):
        run_pnp(t2 * float('nan'), t3, K)
    assert run_pnp(t2[:4], t3[:4], K) == (False, None)
