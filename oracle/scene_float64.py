"""ORACLE (test infrastructure, not product code): float64 restatement of the four scene kernels of
dust3r_b200/csrc/scene_ops.cu -- weighted Procrustes moments, the Weiszfeld focal, the cross-view confidence filter and brute-force
nearest neighbours -- with an error bound for every quantity they return.

The oracle reads exactly what a kernel reads: the fp32 buffers, widened to float64 exactly.  A difference from the kernel is the
kernel's own fp32 arithmetic, and the bounds below cover it.  Notation: u = 2^-24 (one fp32 rounding), u64 = 2^-53,
gamma(n) = n u / (1 - n u), gamma64(n) the same with u64.  The build has no fast math (IEEE `/` and sqrtf, dust3r_b200/build.py);
FMA contraction only removes roundings, so every bound holds for any contraction.  The oracle's own float64 evaluation is one more
summation of the same terms, and is counted wherever it is not negligible against u (the moment and Weiszfeld sums).  Every
constant is derived below; none is fitted to observations.

A value carries (v, e): |fp32 evaluation - v| <= e.  e = 0 means the fp32 evaluation returns v exactly; `_rnd` grants it when
the inputs are exact and v is representable in fp32: a product of two fp32 values is exact in float64, a quotient of two fp32
values that is representable in fp32 is exact too (otherwise it differs from every fp32 value by more than 2^-48 relative), and a
sum with at most one nonzero term is that term.  Everything else takes one rounding: e' = e + u (|v| + e).

Procrustes moments (procrustes_kernel).  17 sums per problem: sum w, sum w x, sum w y, sum w y x^T (w y_a is exact in float64,
times x_b one rounding), sum w |x|^2 (three exact squares, two additions, one product: three roundings).  Each term has at most
3 float64 roundings and any summation order of P terms adds gamma64(P - 1) sum |term|, so the kernel is within
gamma64(P + 3) sum |term| of the exact sum, and so is the oracle's own float64 sum:  bound = 2 gamma64(P + 3) sum |term|.  A
dropped, duplicated or misattributed point moves a moment by about 1 / P of its size: many orders above this.

Rigid registration (scene_ops.rigid_registration, from the moments).  The oracle's R, t, s are the reference's centred-form
Umeyama in float64.  The wrapper forms M = sum w y x^T - sw ym xm^T from uncentred moments, so per element
    dM_ab = dm_ab + |ym_a xm_b| dsw + sw (|xm_b| dym_a + |ym_a| dxm_b + dym_a dxm_b) + 3 u64 (|m_ab| + sw |ym_a| |xm_b|)
(the moment bounds, the centres' bounds dxm = (dSx + |xm| dsw) / (sw - dsw) + u64 |xm| with one rounding for the division, and
the cancellation: two products and a subtraction, 3 u64), and the oracle's centred sums add 2 gamma64(P + 5) sum w |yc_a| |xc_b| (the centre's own error enters only through sum w yc = O(u64): second order,
absorbed by the factor 2).  Both SVDs are backward stable: they factor M + E with |E|_F <= p u64 |M|_F, p = 100 for the 3x3
Householder bidiagonalisation and QR sweeps (the modest p(n) of LAPACK's error bounds), counted once for each side.  The rotation
closest to M in SO(3) moves by |dR|_F <= 2 |dM|_F / (s2 + d s3 - 2 |dM|_F), d = sign det M (the polar-factor bound on the signed
singular values; infinite where the gap is not positive, where R is not unique).  R = U diag(D) V^T: U diag(D) is exact (a sign
flip), and each element of its product with V^T is a three-term dot product of orthonormal rows and columns, so
sum |U_ik| |V_kj| <= 1 and the product adds gamma64(3), once in the wrapper and once in the oracle: 2 gamma64(3).
s = tr(R^T M) / varx: tr(R^T M) is the maximum of tr(Q^T M) over SO(3), so it moves by at most |dM|_* <= sqrt(3) |dM|_F; it is
evaluated as sum S D, a three-term sum with two roundings, on each side: 2 gamma64(2) sum S.  varx = sum w|x|^2 - sw |xm|^2
carries dm16, its centre term and the cancellation 7 u64 (m16 + sw |xm|^2) (|xm|^2: three products and two additions, then
the product with sw and the subtraction: seven roundings of terms bounded by m16 + sw |xm|^2).  t = ym - s R xm propagates dym, ds, dR and dxm, and its own
evaluation -- R xm (three products, two additions), times s, subtracted from ym: five roundings of terms bounded by
|ym| + s |R| |xm| -- adds gamma64(5) on each side: 2 gamma64(5).  The outputs are rounded to fp32: one u each.

Weiszfeld focal (weiszfeld_kernel), one step as a function of the previous fp32 focal f (steps = k against one step fed the
device's steps = k - 1 result).  Per pixel: rays r = x / z (one rounding; 0 where the fp32 quotient is not finite, i.e. NaN or
|x / z| > FLT_MAX), px = (u - cx, v - cy) (one rounding each), num = <r, px>, den = <r, r> (propagated, two products and a sum).
Step 0: weight 1.  Later steps: e = px - f r (a product and a difference), |e| = sqrtf(ex^2 + ey^2): |e - e64| <= |dex| + |dey|
plus gamma(3) (|e| + |dex| + |dey|) for the squares, the sum and the square root; the residual is a difference, so its bound is
absolute.  w = 1 / max(|e|, c) with c = 1e-8f: the clip is 1-Lipschitz, so w lies in [1 / max(|e| + d, c), 1 / max(|e| - d, c)],
plus one rounding.  w num and w den: propagated, one rounding each.  The per-map sums are fp64 (kernel) and float64 (oracle):
2 gamma64(P + 8) sum |term| (8 >= the float64 roundings of one pixel's chain).  f' = A / B: (dA + |f'| dB) / (B - dB) + u64 |f'|,
then one fp32 rounding.  With fp32_sums (the reference, which takes fp32 means in any order) each sum adds gamma(P) sum |term| and
the division by P one more rounding.

clean_pointcloud (clean_kernel), test (i, j) at pixel p: p = T x (four-term dot product, gamma(4) sum |term|), q = K p
(three-term dot product of values known to dp), u = q_x / q_z, v = q_y / q_z (the division bound), then rintf, half to even.  The
test is undecided -- the fp32 evaluation may decide it either way -- where u or v is within its bound of a half-integer, where pz
is within its bound of 0, or where |pz - a depth_j| is within dpz + u |a depth_j|, a = fl32(1 - tol) (its product with an fp32
depth is exact in float64 and rounds once in fp32).  Confidence comparisons and min(c, bad_conf) are exact in fp32 and are never
undecided, and a pixel's result is always c or min(c, bad_conf).  Image i is evaluated against a given set of confidences for the
other images (the device's own final ones for j < i in the tests), so every pixel whose tests are all decided has one exact
expected value.

Nearest neighbours (nn_kernel): d2 = fmaf(dx, dx, fmaf(dy, dy, dz * dz)) with dx = fl(a_x - b_x): each difference rounds once
(its square gains 2 u), the three roundings of the sum of squares add 3 u, so d2 lies within gamma(5) of the exact squared
distance, relatively (distances that are normal fp32 numbers or 0).  The kernel keeps the first strict minimum, so its choice k
satisfies d(k) (1 - gamma(5)) <= d(min) (1 + gamma(5)): d(k) <= d(min) (1 + eps), eps = 2 gamma(5) / (1 - gamma(5)).  Exact fp32
duplicates have identical d2, so among them the lowest index is required.  Non-finite input: a NaN distance never compares below
the running best, so a NaN point is never chosen and a query without any finite distance (a NaN query, or all points NaN) gets 0.
"""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
U64 = 2.0 ** -53
F64 = torch.float64
FLT_MAX = float(np.finfo(np.float32).max)
CLIP = float(np.float32(1e-8))          # the kernel's 1e-8f
SVD_P = 100                             # p(3) of the SVD's backward error, see the docstring


def gamma(n, u=U):
    return n * u / (1 - n * u)


NN_EPS = 2 * gamma(5) / (1 - gamma(5))


def f64(t):
    return torch.as_tensor(t).detach().cpu().to(F64)


def is_f32(v):
    return v == v.float().to(F64)


# ------------------------------------------------------------------------------------------- bounded arithmetic: (value, bound)
def _rnd(v, e, u=U):
    """One rounding of a value known to e; exact (0) when the inputs are exact and v is representable in fp32."""
    exact = (e == 0) & is_f32(v)
    return v, torch.where(exact, torch.zeros_like(e), e + u * (v.abs() + e))


def _mul(a, da, b, db, u=U):
    return _rnd(a * b, da * b.abs() + a.abs() * db + da * db, u)


def _add(a, da, b, db, u=U):
    return _rnd(a + b, da + db, u)


def _sub(a, da, b, db, u=U):
    return _rnd(a - b, da + db, u)


def _div(a, da, b, db, u=U):
    v = a / b
    e = (da + v.abs() * db) / (b.abs() - db)
    e = torch.where(b.abs() > db, e, torch.full_like(e, math.inf))
    e = torch.where((da == 0) & (db == 0), torch.zeros_like(e), e)
    return _rnd(v, e, u)


def _dot(coef, vals, dvals, u=U):
    """sum_k coef_k vals_k of fp32 coefficients (broadcast) and values known to dvals, in any fp32 order / contraction."""
    terms = coef * vals
    prop = (coef.abs() * dvals).sum(-1)
    v = terms.sum(-1)
    single = ((terms != 0).sum(-1) <= 1) & (prop == 0)
    e = prop + gamma(terms.shape[-1], u) * (terms.abs().sum(-1) + prop)
    _, e1 = _rnd(v, torch.zeros_like(v), u)
    return v, torch.where(single, e1, e)


# ------------------------------------------------------------------------------------------------------------ Procrustes
def moments64(x, y, w):
    """(B,P,3), (B,P,3), (B,P) -> the kernel's 17 moments (B,17) and their bounds."""
    x, y, w = f64(x), f64(y), f64(w)
    wy = w[..., None] * y
    terms = torch.cat([w[..., None], w[..., None] * x, wy, (wy[..., :, None] * x[..., None, :]).flatten(-2),
                       (w * (x * x).sum(-1))[..., None]], -1)
    P = x.shape[1]
    return terms.sum(1), 2 * gamma(P + 3, U64) * terms.abs().sum(1)


def umeyama64(x, y, w, compute_scaling=True):
    """Centred-form weighted Umeyama in float64: R (B,3,3), t (B,3), s (B,) and what its bound needs."""
    x, y, w = f64(x), f64(y), f64(w)
    sw = w.sum(1)
    xm, ym = (w[..., None] * x).sum(1) / sw[:, None], (w[..., None] * y).sum(1) / sw[:, None]
    xc, yc = x - xm[:, None], y - ym[:, None]
    M = torch.einsum('bp,bpi,bpj->bij', w, yc, xc)
    Mabs = torch.einsum('bp,bpi,bpj->bij', w, yc.abs(), xc.abs())
    varx = (w * (xc * xc).sum(-1)).sum(1)
    Uu, S, Vh = torch.linalg.svd(M)
    d = torch.sign(torch.linalg.det(Uu @ Vh))
    D = torch.ones_like(S)
    D[:, -1] = d
    R = Uu @ torch.diag_embed(D) @ Vh
    s = (S * D).sum(-1) / varx if compute_scaling else torch.ones_like(sw)
    t = ym - s[:, None] * (R @ xm[..., None])[..., 0]
    P = x.shape[1]
    return dict(R=R, t=t, s=s, M=M, S=S, detM=torch.linalg.det(M), varx=varx, xm=xm, ym=ym, sw=sw,
                dM_own=2 * gamma(P + 5, U64) * Mabs, dvarx_own=2 * gamma(P + 5, U64) * (w * (xc * xc).sum(-1)).sum(1))


def registration64(x, y, w, m=None, dm=None, compute_scaling=True):
    """The oracle's R, t, s and the bounds dR (B,3,3), dt (B,3), ds (B,) of the wrapper's fp32 outputs, from the moments m and
    their bounds dm (the oracle's own when not given)."""
    if m is None:
        m, dm = moments64(x, y, w)
    o = umeyama64(x, y, w, compute_scaling)
    sw, dsw = m[:, 0], dm[:, 0]
    xm, ym = m[:, 1:4] / sw[:, None], m[:, 4:7] / sw[:, None]
    dxm = (dm[:, 1:4] + xm.abs() * dsw[:, None]) / (sw - dsw)[:, None] + U64 * xm.abs()
    dym = (dm[:, 4:7] + ym.abs() * dsw[:, None]) / (sw - dsw)[:, None] + U64 * ym.abs()
    yx = ym.abs()[:, :, None] * xm.abs()[:, None, :]
    dM = (dm[:, 7:16].reshape(-1, 3, 3) + yx * dsw[:, None, None]
          + sw[:, None, None] * (xm.abs()[:, None, :] * dym[:, :, None] + ym.abs()[:, :, None] * dxm[:, None, :]
                                 + dym[:, :, None] * dxm[:, None, :])
          + 3 * U64 * (m[:, 7:16].reshape(-1, 3, 3).abs() + sw[:, None, None] * yx))
    MF = o['M'].flatten(1).norm(dim=1)
    dMF = dM.flatten(1).norm(dim=1) + o['dM_own'].flatten(1).norm(dim=1) + 2 * SVD_P * U64 * MF
    S = o['S']
    dsign = torch.where(o['detM'] < 0, -1.0, 1.0).to(F64)
    gap = S[:, 1] + dsign * S[:, 2] - 2 * dMF
    dRF = torch.where(gap > 0, 2 * dMF / gap, torch.full_like(gap, math.inf))
    R, s = o['R'], o['s']
    dR = dRF[:, None, None] + 2 * gamma(3, U64) + U * (R.abs() + dRF[:, None, None])
    if compute_scaling:
        num = (S * torch.where(torch.arange(3) == 2, dsign[:, None], torch.ones_like(S))).sum(-1)
        dnum = math.sqrt(3) * dMF + 2 * gamma(2, U64) * S.sum(-1)
        varx = o['varx']
        dvarx = (dm[:, 16] + dsw * (xm * xm).sum(-1) + sw * (2 * xm.abs() * dxm + dxm * dxm).sum(-1)
                 + 7 * U64 * (m[:, 16] + sw * (xm * xm).sum(-1)) + o['dvarx_own'])
        ds = (dnum + s.abs() * dvarx) / (varx - dvarx) + U64 * s.abs()
        ds = torch.where(varx > dvarx, ds, torch.full_like(ds, math.inf))
    else:
        ds = torch.zeros_like(s)
    Rx = (R.abs() @ xm.abs()[..., None])[..., 0]
    dt = (dym + ds[:, None] * Rx + s.abs()[:, None] * (dRF[:, None] * xm.abs().sum(-1, keepdim=True)
                                                       + (R.abs() @ dxm[..., None])[..., 0])
          + 2 * gamma(5, U64) * (ym.abs() + s.abs()[:, None] * Rx))
    t = o['t']
    out = dict(R=R, t=t, s=s, dR=dR, dt=dt + U * (t.abs() + dt), ds=ds + U * (s.abs() + ds), gap=gap)
    return out


# -------------------------------------------------------------------------------------------------------------- Weiszfeld
def weiszfeld_step64(pts, pp, W, focal=None, u=U, fp32_sums=False, clip=CLIP, zero_nonfinite=True):
    """One step of weiszfeld_kernel: pts (B,P,3) (the map's pixels row-major, width W), pp (B,2); focal (B,) the previous
    fp32 focal, or None for step 0.  -> (f (B,), df (B,)) for the fp32 result.  u = U64 with fp32_sums=False bounds a float64
    evaluation instead.  clip / zero_nonfinite: deliberate mistakes for the resolution checks."""
    pts, pp = f64(pts), f64(pp)
    B, P, _ = pts.shape
    z0 = torch.zeros((B, P), dtype=F64)
    rays = []
    for k in range(2):
        r = pts[..., k] / pts[..., 2]
        if zero_nonfinite:
            bad = ~(r.abs() <= FLT_MAX) if u == U else ~r.isfinite()
            r = torch.where(bad, z0, r)
        rays.append(_rnd(r, z0, u))
    idx = torch.arange(P)
    grid = [(idx % W).to(F64), torch.div(idx, W, rounding_mode='floor').to(F64)]
    px = [_rnd(grid[k][None] - pp[:, k:k + 1], z0, u) for k in range(2)]
    num = _add(*_mul(*rays[0], *px[0], u), *_mul(*rays[1], *px[1], u), u)
    den = _add(*_mul(*rays[0], *rays[0], u), *_mul(*rays[1], *rays[1], u), u)
    if focal is None:
        wn, wd = num, den
    else:
        fo = f64(focal)[:, None].expand(B, P)
        e = [_sub(*px[k], *_mul(fo, z0, *rays[k], u), u) for k in range(2)]
        n = torch.sqrt(e[0][0] ** 2 + e[1][0] ** 2)
        dn = e[0][1] + e[1][1]
        dn = torch.where((dn == 0) & (n == 0), z0, dn + gamma(3, u) * (n + dn))
        c = torch.full_like(n, clip)
        m = torch.maximum(n, c)
        lo, hi = torch.maximum(n - dn, c), torch.maximum(n + dn, c)
        w = 1 / m
        dw = torch.maximum(1 / lo - w, w - 1 / hi)
        w, dw = w, dw + u * (w + dw)
        wn, wd = _mul(w, dw, *num, u), _mul(w, dw, *den, u)
    sums = []
    for v, e in (wn, wd):
        S, dS = v.sum(1), e.sum(1) + 2 * gamma(P + 8, U64) * v.abs().sum(1)
        if fp32_sums:
            dS = dS + gamma(P) * v.abs().sum(1)
            S, dS = S / P, dS / P
            dS = dS + U * (S.abs() + dS)
        sums.append((S, dS))
    (A, dA), (Bs, dB) = sums
    f = A / Bs
    df = (dA + f.abs() * dB) / (Bs.abs() - dB) + U64 * f.abs()
    df = torch.where(Bs.abs() > dB, df, torch.full_like(df, math.inf))
    return f, df + u * (f.abs() + df)


def weiszfeld64(pts, pp, W, steps=10, u=U64):
    """The whole IRLS in float64 (values only): the focal after `steps` re-weighted steps."""
    f, _ = weiszfeld_step64(pts, pp, W, None, u=u)
    for _ in range(steps):
        f, _ = weiszfeld_step64(pts, pp, W, f, u=u)
    return f


def check_focal(got, f, df):
    """err / bound of fp32 focals against (f, df); a non-finite pattern mismatch is an infinite ratio."""
    got = f64(got)
    if not torch.equal(got.isfinite(), f.isfinite()):
        return math.inf
    ok = f.isfinite()
    err = (got[ok] - f[ok]).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / df[ok])
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------------------- clean_pointcloud
def coef32(tol):
    """The kernel's (1 - tol) as fp32: 1.f - tol with tol an fp32 argument."""
    return float(np.float32(1) - np.float32(tol))


def clean_image64(i, pts, confs, depths, hw, K, T, tol, bad_conf, coef=None, u=U, mutant=None):
    """Image i's new confidences against the given confidences `confs` of every image (confs[i] is image i's input):
    -> (expected (P_i,) float64, undecided (P_i,) bool).  pts / depths per image, flat (P_j,3) / (P_j,); hw [(H, W)];
    K (n,3,3), T (n,4,4) world -> camera.  coef: the fp32 value of (1 - tol) (the kernel's by default).  mutant: 'away' (round
    half away from zero), 'le' (<= in the depth test), 'width' (index image j with image i's width) -- resolution checks."""
    n = len(pts)
    K, T = f64(K), f64(T)
    a = coef32(tol) if coef is None else coef
    x = f64(pts[i]).reshape(-1, 3)
    P = x.shape[0]
    c = f64(confs[i]).reshape(-1).clone()
    und = torch.zeros(P, dtype=torch.bool)
    xh = torch.cat([x, torch.ones((P, 1), dtype=F64)], 1)
    z0 = torch.zeros((P, 4), dtype=F64)
    for j in range(n):
        if j == i:
            continue
        p = [_dot(T[j, r], xh, z0, u) for r in range(3)]
        pv = torch.stack([v for v, _ in p], -1)
        pe = torch.stack([e for _, e in p], -1)
        q = [_dot(K[j, r], pv, pe, u) for r in range(3)]
        uv = [_div(*q[k], *q[2], u) for k in range(2)]
        pz, dpz = p[2]
        Hj, Wj = hw[j]
        rnd = []
        und_uv = torch.zeros(P, dtype=torch.bool)
        for v, e in uv:
            fin = v.isfinite()
            half = (v - torch.floor(v) - 0.5).abs() <= e
            und_uv |= fin & (e > 0) & half
            und_uv |= ~e.isfinite() & ~v.isnan()
            if mutant == 'away':
                rnd.append(torch.sign(v) * torch.floor(v.abs() + 0.5))
            else:
                rnd.append(torch.round(v))          # half to even
        uf, vf = rnd
        und_z = (pz.abs() <= dpz) & (dpz > 0)
        vis = (pz > 0) & (uf >= 0) & (uf < Wj) & (vf >= 0) & (vf < Hj)
        # a rounding that is undecided matters only for a point that may be in front of camera j and near its image
        near = (pz > 0) | und_z
        for (v, _), lim in zip(uv, (Wj, Hj)):
            near &= (v > -1) & (v < lim + 1)
        und_uv &= near
        Wq = hw[i][1] if mutant == 'width' else Wj
        qi = torch.where(vis, vf * Wq + uf, torch.zeros_like(uf)).long().clamp(0, hw[j][0] * hw[j][1] - 1)
        dj, cj = f64(depths[j]).reshape(-1)[qi], f64(confs[j]).reshape(-1)[qi]
        thr = a * dj
        _, dthr = _rnd(thr, torch.zeros_like(thr), u)
        front = (pz <= thr) if mutant == 'le' else (pz < thr)
        und_d = ((pz - thr).abs() <= dpz + dthr) & (dpz + dthr > 0)
        more = c < cj
        und |= und_uv | und_z | (vis & und_d & more)
        cut = vis & front & more
        c = torch.where(cut, torch.clamp(c, max=bad_conf), c)
    return c, und


def clean64(pts, confs, depths, hw, K, T, tol, bad_conf, parallel=False, **kw):
    """The whole filter in float64, sequentially (image i sees the final confidences of images < i) or, with parallel=True, with
    every image reading the input confidences: list of (expected, undecided) per image."""
    cur = [f64(c).reshape(-1) for c in confs]
    out = []
    for i in range(len(pts)):
        given = [confs[j] if parallel or j >= i else cur[j] for j in range(len(pts))]
        c, und = clean_image64(i, pts, given, depths, hw, K, T, tol, bad_conf, **kw)
        cur[i] = c
        out.append((c, und))
    return out


def check_clean(got, pts, confs, depths, hw, K, T, tol, bad_conf, **kw):
    """Compare the fp32 results `got` (per image) with the oracle, image i evaluated against got[j] for j < i and the inputs
    for j > i.  -> (wrong decided pixels, undecided pixels, undecided pixels holding neither possible value, cut pixels)."""
    wrong = und_n = bad_und = cut = 0
    for i in range(len(pts)):
        given = [got[j] if j < i else confs[j] for j in range(len(pts))]
        exp, und = clean_image64(i, pts, given, depths, hw, K, T, tol, bad_conf, **kw)
        g = f64(got[i]).reshape(-1)
        c0 = f64(confs[i]).reshape(-1)
        same = (g == exp) | (g.isnan() & exp.isnan())
        wrong += int((~same & ~und).sum())
        und_n += int(und.sum())
        ok = (g == c0) | (g == torch.clamp(c0, max=bad_conf)) | (g.isnan() & c0.isnan())
        bad_und += int((und & ~ok).sum())
        cut += int((exp != c0).sum())
    return wrong, und_n, bad_und, cut


# --------------------------------------------------------------------------------------------------- nearest neighbours
def _d2(q, p):
    return ((q[:, None, :] - p[None, :, :]) ** 2).sum(-1)


def check_nn(queries, points, got, idx=None, d12=None, chunk=1024):
    """Number of queries whose index `got` the kernel could not have returned: d64(got) > d64(min) (1 + eps), an exact fp32
    duplicate of the chosen point at a lower index, or (no finite distance) anything but 0.  idx: the query rows checked (all by
    default); d12: their (d1, d2) nearest float64 distances from a k-d tree (brute force when not given)."""
    q, p = f64(queries).reshape(-1, 3), f64(points).reshape(-1, 3)
    got = torch.as_tensor(got).cpu().long().reshape(-1)
    if idx is None:
        idx = torch.arange(q.shape[0])
    bad = 0
    for s in range(0, len(idx), chunk):
        rows = idx[s:s + chunk]
        k = got[rows]
        if (k < 0).any() or (k >= p.shape[0]).any():
            return len(idx)
        dk = ((q[rows] - p[k]) ** 2).sum(-1)
        if d12 is None:
            D = _d2(q[rows], p)
            D = torch.where(D.isnan(), torch.full_like(D, math.inf), D)
            dmin = D.min(1).values
        else:
            dmin = d12[s:s + chunk, 0] ** 2
        nofin = ~dmin.isfinite()
        ok = torch.where(nofin, k == 0, dk <= dmin * (1 + NN_EPS))
        # exact duplicates of the chosen point at a lower index
        pk = p[k]
        for r in torch.nonzero(ok & ~nofin)[:, 0].tolist():
            kk = int(k[r])
            if kk and bool((p[:kk] == pk[r]).all(-1).any()):
                ok[r] = False
        bad += int((~ok).sum())
    return bad


def nn64(queries, points):
    """Lowest index among the minimum float64 distances (0 for a query without a finite distance), brute force."""
    q, p = f64(queries).reshape(-1, 3), f64(points).reshape(-1, 3)
    out = []
    for s in range(0, q.shape[0], 1024):
        D = _d2(q[s:s + 1024], p)
        D = torch.where(D.isnan(), torch.full_like(D, math.inf), D)
        out.append(D.argmin(1))          # first minimum
    return torch.cat(out)


def near_tie(queries, points, chunk=1024):
    """Queries whose two nearest float64 distances are within the kernel's eps (either could be returned)."""
    q, p = f64(queries).reshape(-1, 3), f64(points).reshape(-1, 3)
    out = []
    for s in range(0, q.shape[0], chunk):
        D = _d2(q[s:s + chunk], p)
        D = torch.where(D.isnan(), torch.full_like(D, math.inf), D)
        two = D.topk(min(2, p.shape[0]), dim=1, largest=False).values
        out.append(two[:, -1] <= two[:, 0] * (1 + NN_EPS) if p.shape[0] > 1 else torch.zeros(D.shape[0], dtype=torch.bool))
    return torch.cat(out)
