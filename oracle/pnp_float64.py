"""Float64 restatement of the PnP-RANSAC kernels (dust3r_b200/csrc/pnp_core.h, pnp_ops.cu), written independently of them:

  * `sample_indices`: the counter-based draws (SplitMix64's finaliser keyed by seed, hypothesis and draw, duplicates rejected);
  * `epnp`: EPnP (Lepetit, Moreno-Noguer & Fua 2009) as OpenCV's calib3d/src/epnp.cpp computes it, with numpy `eigh` for the
    PCA and for M^T M, `lstsq` for the beta estimates and Gauss-Newton, and an SVD for the rotation (the proper rotation
    U diag(1, 1, det(U V^T)) V^T); `epnp_conditioned` says whether a sample's pose is defined to 1e-10 independently of the
    basis an eigensolver returns for the exactly degenerate null space of a 5-point M (a 10 x 12 matrix), which both sides
    replace by the canonical basis of pnp_core.h;
  * `reproj_err2`: OpenCV's RANSAC callback error -- the projection in float64 in projectPoints' operation order, rounded to
    float32, the squared error in float32 -- and `undecided`, the points whose error lies so close to thr^2 that rounding
    differences in the pose could flip them;
  * `update_num_iters` (RANSACUpdateNumIters) and `ransac_loop`, the sequential loop of RANSACPointSetRegistrator::run.
"""
from __future__ import annotations

import numpy as np

SAMPLE = 5
MAX_DRAWS = 1024
FLAT = 1e-30
DEFAULT_SEED = 0x5DEECE66D
_M64 = (1 << 64) - 1


def _mix64(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def draw(seed, h, k, n):
    z = _mix64((seed + 0x9E3779B97F4A7C15 * (((h << 32) | k) + 1)) & _M64)
    return ((z >> 32) * n) >> 32


def sample_indices(seed, h, n):
    """The 5 indices of hypothesis h in draw order, or None when MAX_DRAWS draws gave fewer than 5 distinct ones."""
    if n == SAMPLE:
        return list(range(SAMPLE))
    out = []
    for k in range(MAX_DRAWS):
        i = draw(seed, h, k, n)
        if i not in out:
            out.append(i)
            if len(out) == SAMPLE:
                return out
    return None


PAIRS = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]


def _pose_from_betas(betas, null, alphas, pw, uv, fx, fy, cx, cy):
    ccs = np.tensordot(betas, null, axes=1).reshape(4, 3)
    pcs = alphas @ ccs
    if pcs[0, 2] < 0:
        ccs, pcs = -ccs, -pcs
    pc0, pw0 = pcs.mean(0), pw.mean(0)
    U, _, Vt = np.linalg.svd((pcs - pc0).T @ (pw - pw0))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt)) or 1.0])
    R = U @ D @ Vt
    t = pc0 - R @ pw0
    Xc = pw @ R.T + t
    err = np.mean(np.hypot(uv[:, 0] - (cx + fx * Xc[:, 0] / Xc[:, 2]), uv[:, 1] - (cy + fy * Xc[:, 1] / Xc[:, 2])))
    return R, t, err


def epnp(pw, uv, fx, fy, cx, cy, null_rotation=None):
    """EPnP on 5 points (float64 (5,3) world, (5,2) pixels) -> (R 3x3, t 3) of least mean reprojection error, or None.
    `null_rotation` (radians) rotates the two null-space vectors of smallest eigenvalue into each other before use."""
    pw, uv = np.asarray(pw, np.float64), np.asarray(uv, np.float64)
    n = len(pw)
    c0 = pw.mean(0)
    d = pw - c0
    lam, E = np.linalg.eigh(d.T @ d)
    lam, E = lam[::-1], E[:, ::-1]
    E = E * np.where(E[np.argmax(np.abs(E), 0), np.arange(3)] < 0, -1.0, 1.0)   # largest component of each direction > 0
    if not (lam[0] > 0) or not np.isfinite(lam[0]):
        return None
    sig = np.where(lam > FLAT * lam[0], np.sqrt(np.maximum(lam, 0) / n), 0.0)
    cws = np.vstack([c0, c0 + sig[:, None] * E.T])
    proj = d @ E
    a = np.divide(proj, sig, out=np.zeros_like(proj), where=sig > 0)
    alphas = np.hstack([1 - a.sum(1, keepdims=True), a])
    M = np.zeros((2 * n, 12))
    for i in range(n):
        for j in range(4):
            M[2 * i, 3 * j] = alphas[i, j] * fx
            M[2 * i, 3 * j + 2] = alphas[i, j] * (cx - uv[i, 0])
            M[2 * i + 1, 3 * j + 1] = alphas[i, j] * fy
            M[2 * i + 1, 3 * j + 2] = alphas[i, j] * (cy - uv[i, 1])
    _, V = np.linalg.eigh(M.T @ M)
    null = V[:, :4].T.copy()           # null[0]: smallest eigenvalue
    if null_rotation is not None:
        c, s = np.cos(null_rotation), np.sin(null_rotation)
        null[0], null[1] = c * null[0] - s * null[1], s * null[0] + c * null[1]
    # the canonical basis of the plane of the two smallest: null[0] along its projection of e = (1, ..., 12)
    e = np.arange(1, 13, dtype=np.float64)
    b0 = null[0] * (null[0] @ e) + null[1] * (null[1] @ e)
    if not np.linalg.norm(b0) > 0:
        return None
    b0 /= np.linalg.norm(b0)
    x = null[0] if abs(b0 @ null[0]) < abs(b0 @ null[1]) else null[1]
    b1 = x - b0 * (b0 @ x)
    null[0], null[1] = b0, b1 / np.linalg.norm(b1)
    dv = [[(null[k].reshape(4, 3)[p] - null[k].reshape(4, 3)[q]) for k in range(4)] for p, q in PAIRS]
    L = np.array([[dv[r][0] @ dv[r][0], 2 * dv[r][0] @ dv[r][1], dv[r][1] @ dv[r][1], 2 * dv[r][0] @ dv[r][2],
                   2 * dv[r][1] @ dv[r][2], dv[r][2] @ dv[r][2], 2 * dv[r][0] @ dv[r][3], 2 * dv[r][1] @ dv[r][3],
                   2 * dv[r][2] @ dv[r][3], dv[r][3] @ dv[r][3]] for r in range(6)])
    rho = np.array([np.sum((cws[p] - cws[q]) ** 2) for p, q in PAIRS])
    best = None
    for variant, cols in ((1, [0, 1, 3, 6]), (2, [0, 1, 2]), (3, [0, 1, 2, 3, 4])):
        x = np.linalg.lstsq(L[:, cols], rho, rcond=None)[0]
        b = np.zeros(4)
        if variant == 1:
            r = np.sqrt(abs(x[0]))
            b[0], b[1:] = r, (-1 if x[0] < 0 else 1) * x[1:] / r
        else:
            b[0] = np.sqrt(abs(x[0]))
            b[1] = (np.sqrt(-x[2]) if x[2] < 0 else 0.0) if x[0] < 0 else (np.sqrt(x[2]) if x[2] > 0 else 0.0)
            if x[1] < 0:
                b[0] = -b[0]
            if variant == 3:
                b[2] = x[3] / b[0]
        for _ in range(5):   # Gauss-Newton on the six distances
            B = np.array([b[0] ** 2, b[0] * b[1], b[1] ** 2, b[0] * b[2], b[1] * b[2], b[2] ** 2, b[0] * b[3], b[1] * b[3],
                          b[2] * b[3], b[3] ** 2])
            J = np.stack([2 * L[:, 0] * b[0] + L[:, 1] * b[1] + L[:, 3] * b[2] + L[:, 6] * b[3],
                          L[:, 1] * b[0] + 2 * L[:, 2] * b[1] + L[:, 4] * b[2] + L[:, 7] * b[3],
                          L[:, 3] * b[0] + L[:, 4] * b[1] + 2 * L[:, 5] * b[2] + L[:, 8] * b[3],
                          L[:, 6] * b[0] + L[:, 7] * b[1] + L[:, 8] * b[2] + 2 * L[:, 9] * b[3]], 1)
            b = b + np.linalg.lstsq(J, rho - L @ B, rcond=None)[0]
        with np.errstate(all='ignore'):
            R, t, err = _pose_from_betas(b, null, alphas, pw, uv, fx, fy, cx, cy)
        if np.isfinite(err) and np.all(np.isfinite(R)) and np.all(np.isfinite(t)) and (best is None or err < best[2]):
            best = (R, t, err)
    return None if best is None else (best[0], best[1])


def epnp_conditioned(pw, uv, fx, fy, cx, cy, kappa=1e5):
    """(pose or None, well-conditioned).  Well-conditioned when the world points are not (nearly) planar, the pose does not depend on the basis an eigensolver returns
    for the degenerate null space (rotating it changes nothing beyond 1e-12) and a relative perturbation of 1e-12 of the
    inputs moves the pose by at most kappa * 1e-12: then float64 rounding (1.1e-16) cannot move it by more than about
    kappa * 1e-16 = 1e-11."""
    pw, uv = np.asarray(pw, np.float64), np.asarray(uv, np.float64)
    rng = np.random.default_rng(12345)
    flat = lambda p: np.hstack([p[0].ravel(), p[1]])
    try:
        with np.errstate(all='ignore'):
            a = epnp(pw, uv, fx, fy, cx, cy)
            b = epnp(pw, uv, fx, fy, cx, cy, null_rotation=0.6)
            c = epnp(pw * (1 + 1e-12 * rng.standard_normal(pw.shape)), uv * (1 + 1e-12 * rng.standard_normal(uv.shape)),
                     fx, fy, cx, cy)
    except np.linalg.LinAlgError:
        return None, False
    if a is None or b is None or c is None:
        return a, False
    lam = np.linalg.eigvalsh((pw - pw.mean(0)).T @ (pw - pw.mean(0)))
    if not lam[0] > 1e-8 * lam[2]:
        return a, False   # (near-)planar sample: eigensolvers' PCA directions differ by ~1e-16 lam_max / lam_min
    scale = max(1.0, np.max(np.abs(flat(a))))
    return a, bool(np.max(np.abs(flat(a) - flat(b))) <= 1e-12 * scale and np.max(np.abs(flat(a) - flat(c))) <= kappa * 1e-12 * scale)


def reproj_err2(R, t, fx, fy, cx, cy, pts3d, pts2d):
    """float32 squared reprojection error of every correspondence (pts3d float32 (n,3), pts2d float32 (n,2))."""
    R, t = np.asarray(R, np.float64), np.asarray(t, np.float64)
    X, Y, Z = (pts3d[:, k].astype(np.float64) for k in range(3))
    x = R[0, 0] * X + R[0, 1] * Y + R[0, 2] * Z + t[0]
    y = R[1, 0] * X + R[1, 1] * Y + R[1, 2] * Z + t[1]
    z = R[2, 0] * X + R[2, 1] * Y + R[2, 2] * Z + t[2]
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        iz = np.where(z != 0, 1.0 / np.where(z != 0, z, 1.0), 1.0)
        pu = (x * iz * fx + cx).astype(np.float32)
        pv = (y * iz * fy + cy).astype(np.float32)
        du, dv = pts2d[:, 0] - pu, pts2d[:, 1] - pv
        return du * du + dv * dv


def thr2_of(threshold):
    return np.float32(float(threshold) * float(threshold))


def undecided(R, t, fx, fy, cx, cy, pts3d, pts2d, threshold, rel=1e-9):
    """Points whose inlier decision a relative pose perturbation of `rel` or one float32 rounding of the projection could flip:
    |err - thr^2| <= 2 (|e| + u) (rel * (|u| + |v| + |f|) + 2 ulp(u)) + ulp(thr^2), with |e| the error's length."""
    err = reproj_err2(R, t, fx, fy, cx, cy, pts3d, pts2d).astype(np.float64)
    mag = np.abs(pts2d.astype(np.float64)).max(1) + max(abs(fx), abs(fy)) + max(abs(cx), abs(cy))
    delta = rel * mag + 2 * np.spacing(np.float32(mag)).astype(np.float64)
    e = np.sqrt(np.abs(err))
    thr2 = float(thr2_of(threshold))
    bound = 2 * (e + delta) * delta + float(np.spacing(np.float32(thr2)))
    return np.abs(err - thr2) <= bound


def update_num_iters(p, ep, model_points, max_iters):
    """calib3d/src/ptsetreg.cpp: RANSACUpdateNumIters."""
    p, ep = min(max(p, 0.0), 1.0), min(max(ep, 0.0), 1.0)
    num = max(1.0 - p, np.finfo(np.float64).tiny)
    denom = 1.0 - float(np.power(1.0 - ep, float(model_points)))
    if denom < np.finfo(np.float64).tiny:
        return 0
    num, denom = float(np.log(num)), float(np.log(denom))
    return max_iters if denom >= 0 or -num >= max_iters * (-denom) else int(np.rint(num / denom))


def ransac_loop(counts_of, n, confidence, max_iters):
    """The sequential loop: counts_of(h) -> inlier count of hypothesis h (< 0: invalid).  Returns (best h or -1, its count,
    hypotheses evaluated)."""
    best, best_count, niters = -1, 0, max(max_iters, 1)
    h = 0
    while h < niters:
        c = counts_of(h)
        if n == SAMPLE:
            c = SAMPLE if c >= 0 else -1
        if c > max(best_count, SAMPLE - 1):
            best, best_count = h, c
            niters = 1 if n == SAMPLE else update_num_iters(confidence, (n - c) / n, SAMPLE, niters)
        if n == SAMPLE:
            niters = 1
        h += 1
    return best, best_count, h


def hypothesis(pts2d, pts3d, fx, fy, cx, cy, threshold, seed, h):
    """(indices or None, (R, t) or None, count (-1 when invalid)) of hypothesis h, all in float64 from the float32 points."""
    idx = sample_indices(seed, h, len(pts2d))
    if idx is None:
        return None, None, -1
    pose = epnp(pts3d[idx].astype(np.float64), pts2d[idx].astype(np.float64), fx, fy, cx, cy)
    if pose is None:
        return idx, None, -1
    return idx, pose, int(np.sum(reproj_err2(*pose, fx, fy, cx, cy, pts3d, pts2d) <= thr2_of(threshold)))


def ransac(pts2d, pts3d, fx, fy, cx, cy, threshold, confidence=0.9999, max_iters=10_000, seed=DEFAULT_SEED):
    """The whole loop from the oracle's own hypotheses: (best, count, evaluated, pose or None, inlier mask)."""
    pts2d, pts3d = np.asarray(pts2d, np.float32), np.asarray(pts3d, np.float32)
    poses = {}

    def counts_of(h):
        _, pose, c = hypothesis(pts2d, pts3d, fx, fy, cx, cy, threshold, seed, h)
        poses[h] = pose
        return c
    best, count, evaluated = ransac_loop(counts_of, len(pts2d), confidence, max_iters)
    if best < 0:
        return best, count, evaluated, None, np.zeros(len(pts2d), bool)
    pose = poses[best]
    mask = (np.ones(len(pts2d), bool) if len(pts2d) == SAMPLE else
            reproj_err2(*pose, fx, fy, cx, cy, pts3d, pts2d) <= thr2_of(threshold))
    return best, count, evaluated, pose, mask


def synth_problem(n, inlier_ratio, noise_px=0.0, seed=0, planar=False, behind=0.0, W=640, H=480, f=500.0):
    """A PnP problem with known pose: world points seen by a camera (fx = fy = f, principal point at the centre), pixels with
    Gaussian noise for the inliers and uniform ones for the outliers; `behind` the share of outliers put behind the camera.
    Returns (pts2d float32 (n,2), pts3d float32 (n,3), K float64 3x3, R, t (world -> camera), inlier bool (n,))."""
    rng = np.random.default_rng(seed)
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1.0]])
    ang = rng.normal(size=3) * 0.3
    th = np.linalg.norm(ang)
    k = ang / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    t = rng.normal(size=3) * 0.5
    uv = rng.uniform([0, 0], [W, H], size=(n, 2))
    depth = rng.uniform(2.0, 8.0, size=n)
    if planar:   # points on the plane z_cam = 5 + 0.3 x_cam (a tilted wall)
        xn = (uv[:, 0] - K[0, 2]) / f
        depth = 5.0 / (1 - 0.3 * xn)
    Xc = np.stack([(uv[:, 0] - K[0, 2]) / f * depth, (uv[:, 1] - K[1, 2]) / f * depth, depth], 1)
    pts3d = (Xc - t) @ R            # world = R^T (Xc - t)
    inl = rng.uniform(size=n) < inlier_ratio
    pts2d = uv + rng.normal(size=(n, 2)) * noise_px
    out = ~inl
    pts2d[out] = rng.uniform([0, 0], [W, H], size=(int(out.sum()), 2))
    if behind > 0:
        back = out & (rng.uniform(size=n) < behind)
        Xb = Xc[back] * np.array([1, 1, -1.0])
        pts3d[back] = (Xb - t) @ R
    return pts2d.astype(np.float32), pts3d.astype(np.float32), K, R, t, inl
