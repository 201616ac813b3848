"""ORACLE (test infrastructure, not product code): float64 restatement of what the fused alignment kernels
(dust3r_b200/csrc/align_stream.cu, align_step.cu, align_common.cuh) compute, with an error bound for every element.

The oracle reads exactly what a kernel reads -- the packed observations (q, w) with the loss coefficient folded into w,
the fp32 parameters in the `small` layout and the fp32 log-depths -- widened to float64 exactly.  So a difference from
the kernel is the kernel's own fp32 arithmetic, and the bound below has to cover it element by element.

Notation (u = 2^-24, one fp32 rounding; every norm |.| of a vector is its 1-norm, which bounds the 2-norm):
  per image i, pixel p:   X = R c + T,  Y = X - T = R c,  c = (d (u-cx)/fx, d (v-cy)/fy, d),  d = exp(logd)
                          C = (d (|u|+|cx|)/fx, d (|v|+|cy|)/fy, d): the magnitudes the rounding of c sees
  per entry e (edge, side) of image i:   r = X - (M q + t),  M = s R_e diag(adapt),  t = s T_e
      l1: term = w |r|,    G = w r / |r|            l2: term = w |r|^2,   G = 2 w r
  dL/dlogd(p) = sum_e G_e,p . Y_p

Residual error (absolute, the reason no relative tolerance can work):
  dX  = c3 u (sum_ab |R_ab| C_b + |T|) + eps_exp |Y|          c3 = 16: d, (u-cx), 1/fx, R (from the quaternion),
                                                               the three-term FMA, and the fp32 cx / 1/fx themselves
  dr  = dX + c3 u (sum_ab |M_ab q_b| + |t|)                    M carries s = exp(.) exp(log b - mean), R and adapt
  kappa:  l1: min(2 dr / |r|, 2)   (direction of G)           l2: 2 dr   (|G| = 2 w |r|)
  eps_exp: streaming kernel __expf (ex2.approx), CUDA documents 2 + floor(|1.173 x|) ulp; general kernel expf, 2 ulp.
           One ulp of the result is at most 2^-23 of it.  eps_rsqrt = 2^-22.9, the PTX bound of rsqrt.approx.f32.

Per-pixel gradient (kernel gd = sum over the image's deg entries of G, then . Y):
  |gd - gd64| <= sum_e |Y| ( |G| (c1 u + eps_rsqrt) + w kappa ) + sum_e |G| dX + |gd64| c2 u,
  c1 = 2 (deg + 6) (the chain of deg additions of G, the 3-term dot and the products), c2 = 4.

Per-entry loss (E x 2) and total loss: every term is >= 0.
  |L_e - L64_e| <= 2 k_e u sum_p term + sum_p w dterm + n_e 2^-41 + u |L64_e|
      dterm = l1: dr + |r| (eps_rsqrt + 4u);  l2: 2 |r| dr + dr^2 + 4u |r|^2
  total: sum of the entry bounds + 2 (ceil(2E/256) + 13) u sum_e L_e  (the last CTA's block sum).

Small-parameter gradients.  The kernel sums, per entry, S = sum_p G (x) q (9) and sum_p G (3), and per image
sum_p G (x) c (general kernel) or sum_p G (x) Y, then times R (streaming kernel), plus sum_p G; the last CTA maps these
sums linearly to the gradients.  With J = d(M, t)/d(edge parameters) and J = d(R K K0^-1, T)/d(image parameters)
(K = [[1/fx, 0, -cx/fx], [0, 1/fy, -cy/fy], [0, 0, 1]], K0 = K at the current value, so that X = R K m + T with m
independent of the parameters and sum G (x) m = S K^-T), the gradient is g_theta = -/+ sum_k J_k,theta S_k, and
  |g - g64| <= sum_k |J_k,theta| ( (2 k u + eps_rsqrt) H_k + Hkappa_k + n_partials_k 2^-41 )
  H_k      = sum_p |G_a| |q_b|   (entries)  or  2 sum_p |G_a| |C|   (images, 2 covers the streaming kernel's S R)
  Hkappa_k = sum_p w kappa |q_b|            or  2 sum_p (w kappa + c3 u |G|) |C|
  k = longest fp32 summation chain before the fixed-point atomics:
      streaming: 3 (slots of a lane) + 1 (pixel pair) + 5 (warp transpose) + the warp's items of one image kept in
                 one window + 2 (products)
      general:   8 (pixels of a thread) + 5 (butterfly) + 8 (warps of the CTA) + 2 (products) = 23
  n_partials = fix_add calls feeding one accumulator, counted from the item table (streaming: one per warp run of the
      image, one per item when the image's entries spill the window) or the image's CTAs (general kernel).
  The log-scale of edge e is coupled to every edge through the mean (norm_pw_scale): its bound adds 1/E times the sum
  of every edge's log-scale bound, the fp32 block sum of the mean ((ceil(E/256) + 13 + 2) u mean_e A_e, A_e = the
  edge's sum_k |J_k| H_k) and the rounding of the subtraction (u A_e).  quat_backward forms the quaternion gradient
  before projecting it onto |q| = 1, so the quaternion entries add C_Q u (|g_u| + |qhat| sum |g_u|) with g_u the
  unprojected gradient's magnitude (dR/dq at fixed |q|, times s adapt for edges), C_Q = 8.  The last term, sum_k |J| n_partials 2^-41, is the fixed-point quantisation.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional

import numpy as np
import torch

from .align_oracle import pw_transforms, quat_xyzw_to_rotmat, signed_expm1

U = 2.0 ** -24
EPS_RSQRT = 2.0 ** -22.9
C1_EXTRA, C2, C3 = 6, 4.0, 16.0
FIX_Q = 2.0 ** -41                    # half a quantum of the 2^40 fixed-point accumulators
SLOT_PX = 64
F64 = torch.float64


@dataclass
class Scene64:
    """What one alignment launch reads, in float64.  Entries are in the engine's CSR order (by image, then edge)."""
    imshapes: list
    edges: list
    ent_img: np.ndarray
    ent_edge: np.ndarray
    ent_side: np.ndarray
    q: List[torch.Tensor]             # per entry (P_img, 3)
    w: List[torch.Tensor]             # per entry (P_img,), loss coefficient folded in
    logd: List[torch.Tensor]          # per image (P,)
    small: torch.Tensor               # (11n + 10E,)
    dist: str = 'l1'
    kernel: str = 'stream'
    tied_focal: bool = True
    norm_pw_scale: bool = True
    base_scale: float = 0.5
    pw_break: float = 20.0
    focal_break: float = 20.0
    n_partials_ent: Optional[np.ndarray] = None    # per entry
    n_partials_img: Optional[np.ndarray] = None    # per image
    chain_ent: Optional[np.ndarray] = None         # summation chain k per entry
    chain_img: Optional[np.ndarray] = None

    @property
    def n(self):
        return len(self.imshapes)

    @property
    def E(self):
        return len(self.edges)

    def offsets(self):
        n, E = self.n, self.E
        return dict(poses=0, focals=7 * n, pp=9 * n, pw=11 * n, adapt=11 * n + 8 * E, total=11 * n + 10 * E)


def entry_order(n, edges):
    """The engine's CSR: for every image, its (edge, side) entries sorted by edge."""
    img, edge, side = [], [], []
    for i in range(n):
        for e, (a, b) in enumerate(edges):
            for s, x in ((0, a), (1, b)):
                if x == i:
                    img.append(i), edge.append(e), side.append(s)
    return np.array(img), np.array(edge), np.array(side)


# ---------------------------------------------------------------------------------------------- chains and partials
def stream_partials(items, warp_ptr, n, deg, window):
    """(fix_add calls per entry accumulator of every image, per image accumulator, longest window chain per image) of the
    streaming kernel, from its item table and warp split (engine.build_stream_items)."""
    runs = np.zeros(n, dtype=np.int64)
    n_items = np.zeros(n, dtype=np.int64)
    chain = np.zeros(n, dtype=np.int64)
    for w in range(len(warp_ptr) - 1):
        prev, length = -1, 0
        for it in range(int(warp_ptr[w]), int(warp_ptr[w + 1])):
            img = int(items['img'][it])
            n_items[img] += 1
            if img != prev:
                runs[img] += 1
                length = 0
            length += 1
            chain[img] = max(chain[img], length if deg[img] <= window else 1)
            prev = img
    ent = np.where(np.asarray(deg) <= window, runs, n_items)
    return ent, runs, chain


def set_chains(sc: Scene64, *, chunk_px=None, items=None, warp_ptr=None, window=None):
    """Fills n_partials_* and chain_* for the scene's kernel (see the module docstring)."""
    n = sc.n
    deg = np.bincount(sc.ent_img, minlength=n)
    areas = np.array([h * w for h, w in sc.imshapes])
    if sc.kernel == 'stream':
        pe, pi, run = stream_partials(items, warp_ptr, n, deg, window)
        k = 3 + 1 + 5 + run + 2
    else:
        pe = pi = (areas + chunk_px - 1) // chunk_px
        k = np.full(n, 8 + 5 + 8 + 2)
    sc.n_partials_img, sc.chain_img = pi.astype(np.float64), k.astype(np.float64)
    sc.n_partials_ent, sc.chain_ent = pe[sc.ent_img].astype(np.float64), k[sc.ent_img].astype(np.float64)


# ---------------------------------------------------------------------------------------------- construction
def scene_from_engine(eng) -> Scene64:
    """Reads the packed observations, the parameters and the item table of an AlignEngine (engine.py)."""
    from dust3r_b200.cloud_opt.engine import ITEM
    obs = eng.obs.detach().double().cpu()
    ent_ptr = eng._ent_ptr.cpu().numpy()
    ent_edge = eng._ent_edge.cpu().numpy()
    ent_off = eng._ent_obs_off.cpu().numpy()
    coef = eng._ent_coef.cpu().numpy().astype(np.float64)
    edge_ent = eng._edge_ent.cpu().numpy()
    n, E = eng.n, eng.E
    ent_img = np.repeat(np.arange(n), np.diff(ent_ptr))
    ent_side = np.array([0 if edge_ent[ent_edge[k], 0] == k else 1 for k in range(2 * E)])
    q, w = [], []
    for k in range(2 * E):
        P = eng.areas[ent_img[k]]
        o = int(ent_off[k])
        if eng.kernel == 'stream':
            ns = (P + SLOT_PX - 1) // SLOT_PX
            slab = obs[o:o + ns * SLOT_PX].reshape(ns, 2, 32, 4)
            xy, zw = slab[:, 0], slab[:, 1]
            x, y = xy[..., 0:2].reshape(-1), xy[..., 2:4].reshape(-1)
            z, ww = zw[..., 0:2].reshape(-1), zw[..., 2:4].reshape(-1)
            q.append(torch.stack((x, y, z), -1)[:P])
            w.append(ww[:P])
        else:
            rows = obs[o:o + P]
            q.append(rows[:, :3].clone())
            w.append(rows[:, 3] * coef[k])
    logd_all = eng.logd.detach().double().cpu()
    logd = [logd_all[int(eng.pix_off[i]):int(eng.pix_off[i]) + eng.areas[i]].clone() for i in range(n)]
    sc = Scene64(imshapes=list(eng.imshapes), edges=list(eng.edges), ent_img=ent_img, ent_edge=ent_edge, ent_side=ent_side,
                 q=q, w=w, logd=logd, small=eng.small.detach().double().cpu(), dist=eng.dist, kernel=eng.kernel,
                 tied_focal=eng.tied_focal, norm_pw_scale=eng.norm_pw_scale, base_scale=eng.base_scale,
                 pw_break=eng.pw_break, focal_break=eng.focal_break)
    if eng.kernel == 'stream':
        items = eng._items.cpu().numpy().view(ITEM)
        set_chains(sc, items=items, warp_ptr=eng._warp_item_ptr.cpu().numpy(), window=eng.stream_window)
    else:
        set_chains(sc, chunk_px=eng.chunk_px)
    return sc


def scene_from_problem(prob, P, kernel='stream', fx_and_fy=False, **chains) -> Scene64:
    """A Scene64 of an oracle AlignProblem (align_oracle.py) and its parameters, every value in float64; w = the
    problem's weight times the float64 loss coefficient (1 / total area per side, or 1 / (P E) per edge)."""
    n, E = prob.n_imgs, len(prob.edges)
    ent_img, ent_edge, ent_side = entry_order(n, prob.edges)
    areas = [h * w for h, w in prob.imshapes]
    tot = [sum(areas[i] for i, j in prob.edges), sum(areas[j] for i, j in prob.edges)]
    q, w = [], []
    for img, e, s in zip(ent_img, ent_edge, ent_side):
        coef = 1.0 / tot[s] if prob.variant == 'stacked' else 1.0 / (areas[img] * E)
        q.append((prob.pred_i if s == 0 else prob.pred_j)[e].double())
        w.append((prob.weight_i if s == 0 else prob.weight_j)[e].double() * coef)
    f = P['im_focals'].double().reshape(n, -1).expand(n, 2)
    small = torch.cat([P['im_poses'].double().reshape(-1), f.reshape(-1), P['im_pp'].double().reshape(-1),
                       P['pw_poses'].double().reshape(-1), P['pw_adaptors'].double().reshape(-1)])
    sc = Scene64(imshapes=list(prob.imshapes), edges=list(prob.edges), ent_img=ent_img, ent_edge=ent_edge, ent_side=ent_side,
                 q=q, w=w, logd=[t.double() for t in P['im_depthmaps']], small=small, dist=prob.dist, kernel=kernel,
                 tied_focal=not fx_and_fy, norm_pw_scale=prob.norm_pw_scale, base_scale=prob.base_scale,
                 pw_break=prob.pw_break, focal_break=prob.focal_break)
    if chains:
        set_chains(sc, **chains)
    return sc


# ---------------------------------------------------------------------------------------------- the float64 objective
def _split(sc: Scene64, small):
    o = sc.offsets()
    n, E = sc.n, sc.E
    f = small[o['focals']:o['pp']].reshape(n, 2)
    if sc.tied_focal:
        f = f[:, :1].expand(n, 2)
    return (small[o['poses']:o['focals']].reshape(n, 7), f, small[o['pp']:o['pw']].reshape(n, 2),
            small[o['pw']:o['adapt']].reshape(E, 8), small[o['adapt']:].reshape(E, 2))


def _pixel_grid(H, W):
    v, u = torch.meshgrid(torch.arange(H, dtype=F64), torch.arange(W, dtype=F64), indexing='ij')
    return u.reshape(-1), v.reshape(-1)


def image_geometry(sc: Scene64, small, logd):
    """Per image: R (3,3), T (3,), K (3,3), and per pixel X, Y, C (magnitudes), d."""
    poses, f, pp, _, _ = _split(sc, small)
    R = quat_xyzw_to_rotmat(poses[:, :4])
    T = signed_expm1(poses[:, 4:7])
    ef = (f / sc.focal_break).exp()
    out = []
    for i, (H, W) in enumerate(sc.imshapes):
        u, v = _pixel_grid(H, W)
        cx, cy = W / 2 + 10 * pp[i, 0], H / 2 + 10 * pp[i, 1]
        d = logd[i].exp()
        c = torch.stack((d * (u - cx) / ef[i, 0], d * (v - cy) / ef[i, 1], d), -1)
        Cm = torch.stack((d * (u.abs() + cx.abs()) / ef[i, 0], d * (v.abs() + cy.abs()) / ef[i, 1], d), -1)
        Y = c @ R[i].T
        out.append(dict(R=R[i], T=T[i], c=c, Cm=Cm, d=d, Y=Y, X=Y + T[i]))
    return out


def edge_transforms(sc: Scene64, small):
    _, _, _, pw, ad = _split(sc, small)
    prob = SimpleNamespace(norm_pw_scale=sc.norm_pw_scale, base_scale=sc.base_scale, pw_break=sc.pw_break)
    sR, sT, adapt = pw_transforms(prob, pw, ad)
    return sR * adapt[:, None, :], sT          # M = s R diag(adapt), t = s T


def loss64(sc: Scene64, small, logd):
    """The objective as the kernels define it: sum over entries and pixels of w * dist(r); differentiable."""
    geo = image_geometry(sc, small, logd)
    M, t = edge_transforms(sc, small)
    loss = 0
    for k in range(len(sc.q)):
        e, i = sc.ent_edge[k], sc.ent_img[k]
        r = geo[i]['X'] - (sc.q[k] @ M[e].T + t[e])
        loss = loss + ((r.norm(dim=-1) if sc.dist == 'l1' else r.square().sum(-1)) * sc.w[k]).sum()
    return loss


def small_grad64(sc: Scene64):
    """dL/d(small) by autograd in float64, laid out like the kernel's small_grad (tied focals: both slots hold the total)."""
    small = sc.small.clone().requires_grad_(True)
    loss = loss64(sc, small, sc.logd)
    (g,) = torch.autograd.grad(loss, small)
    if sc.tied_focal:
        o = sc.offsets()
        gf = g[o['focals']:o['pp']].reshape(sc.n, 2)
        gf[:, :] = gf[:, :1].clone()
    return float(loss.detach()), g.detach()


# ---------------------------------------------------------------------------------------------- per-term quantities
def eps_exp(sc: Scene64, ld):
    if sc.kernel == 'stream':
        return (2 + torch.floor((1.173 * ld).abs())) * 2.0 ** -23
    return torch.full_like(ld, 2 * 2.0 ** -23)


def terms(sc: Scene64):
    """Every (entry, pixel) quantity the bounds need, plus the per-pixel gradient in float64."""
    small = sc.small
    geo = image_geometry(sc, small, sc.logd)
    M, t = edge_transforms(sc, small)
    n = sc.n
    deg = np.bincount(sc.ent_img, minlength=n)
    gd = [torch.zeros(h * w, dtype=F64) for h, w in sc.imshapes]
    gd_bound = [torch.zeros(h * w, dtype=F64) for h, w in sc.imshapes]
    per = []
    for i, g in enumerate(geo):
        Ya = g['Y'].abs().sum(-1)
        g['Ya'] = Ya
        g['Cn'] = g['Cm'].sum(-1)
        g['dX'] = C3 * U * ((g['Cm'] @ g['R'].abs().T).sum(-1) + g['T'].abs().sum()) + eps_exp(sc, sc.logd[i]) * Ya
    for k in range(len(sc.q)):
        e, i = int(sc.ent_edge[k]), int(sc.ent_img[k])
        g = geo[i]
        q, w = sc.q[k], sc.w[k]
        A = q @ M[e].T + t[e]
        r = g['X'] - A
        rn = r.norm(dim=-1)
        Mq = (q.abs() @ M[e].abs().T).sum(-1)
        dr = g['dX'] + C3 * U * (Mq + t[e].abs().sum())
        if sc.dist == 'l1':
            safe = torch.where(rn > 0, rn, torch.ones_like(rn))
            G = torch.where(rn[:, None] > 0, w[:, None] * r / safe[:, None], torch.zeros_like(r))
            term = w * rn
            kappa = torch.where(rn > 0, torch.clamp(2 * dr / safe, max=2.0), torch.full_like(rn, 2.0))
            dterm = w * (dr + rn * (EPS_RSQRT + 4 * U))
            eps_g = EPS_RSQRT
        else:
            G = 2 * w[:, None] * r
            term = w * rn.square()
            kappa = 2 * dr
            dterm = w * (2 * rn * dr + dr.square() + 4 * U * rn.square())
            eps_g = 0.0
        Gn = G.abs().sum(-1)
        contrib = (G * g['Y']).sum(-1)
        gd[i] += contrib
        c1 = 2 * (deg[i] + C1_EXTRA)
        gd_bound[i] += g['Ya'] * (Gn * (c1 * U + eps_g) + w.abs() * kappa) + Gn * g['dX']
        per.append(dict(e=e, i=i, r=r, G=G, Gn=Gn, term=term, dterm=dterm, kappa=kappa, contrib=contrib, q=q, w=w))
    for i in range(n):
        gd_bound[i] += C2 * U * gd[i].abs()
    return dict(geo=geo, per=per, gd=gd, gd_bound=gd_bound, M=M, t=t)


def loss_bounds(sc: Scene64, T):
    """(entry losses (2E,) in float64, their bounds, total loss, its bound), entries in CSR order."""
    L = torch.stack([p['term'].sum() for p in T['per']])
    Lb = torch.stack([2 * sc.chain_ent[k] * U * p['term'].sum() + p['dterm'].sum() for k, p in enumerate(T['per'])])
    Lb = Lb + torch.as_tensor(sc.n_partials_ent) * FIX_Q + U * L.abs()
    k_tot = math.ceil(len(L) / 256) + 13
    return L, Lb, float(L.sum()), float(Lb.sum() + 2 * k_tot * U * L.abs().sum())


# ---------------------------------------------------------------------------------------------- small-parameter bound
def _edge_jacobian(sc: Scene64):
    """(E, 12, 10): d(M (9), t (3)) / d(pw pose 8, adaptors 2) per edge, the normalisation's mean over edges held fixed
    (its coupling is added separately)."""
    o = sc.offsets()
    pw = sc.small[o['pw']:o['adapt']].reshape(sc.E, 8)
    ad = sc.small[o['adapt']:].reshape(sc.E, 2)
    mean_sigma = pw[:, 7].mean()

    def f(x):
        p8, a2 = x[:8], x[8:]
        R = quat_xyzw_to_rotmat(p8[:4])
        T = signed_expm1(p8[4:7])
        s = p8[7].exp()
        a3 = torch.stack((a2[0], a2[0], a2[1]))
        if sc.norm_pw_scale:
            s = s * (math.log(sc.base_scale) - mean_sigma).exp()
            a3 = a3 - a3.mean()
        a3 = (a3 / sc.pw_break).exp()
        return torch.cat(((s * R * a3[None, :]).reshape(-1), s * T))
    x = torch.cat((pw, ad), 1)
    return torch.func.vmap(torch.func.jacfwd(f))(x)


def _image_jacobian(sc: Scene64):
    """(n, 12, 11): d(R K K0^-1 (9), T (3)) / d(pose 7, focal 2, pp 2) per image; with tied focals column 7 is the
    derivative by the shared focal and column 8 repeats it."""
    o = sc.offsets()
    poses = sc.small[o['poses']:o['focals']].reshape(sc.n, 7)
    foc = sc.small[o['focals']:o['pp']].reshape(sc.n, 2)
    pp = sc.small[o['pp']:o['pw']].reshape(sc.n, 2)
    HW = torch.tensor(sc.imshapes, dtype=F64)

    def K_of(f2, p2, hw):
        fx, fy = (f2 / sc.focal_break).exp().unbind()
        cx, cy = hw[1] / 2 + 10 * p2[0], hw[0] / 2 + 10 * p2[1]
        z = torch.zeros((), dtype=F64)
        one = torch.ones((), dtype=F64)
        return torch.stack((torch.stack((1 / fx, z, -cx / fx)), torch.stack((z, 1 / fy, -cy / fy)), torch.stack((z, z, one))))

    def f(x, hw, K0inv):
        p7, f2, p2 = x[:7], x[7:9], x[9:11]
        if sc.tied_focal:
            f2 = torch.stack((f2[0], f2[0]))
        R = quat_xyzw_to_rotmat(p7[:4])
        return torch.cat(((R @ K_of(f2, p2, hw) @ K0inv).reshape(-1), signed_expm1(p7[4:7])))
    K0inv = torch.stack([torch.linalg.inv(K_of(foc[i], pp[i], HW[i])) for i in range(sc.n)])
    J = torch.func.vmap(torch.func.jacfwd(f))(torch.cat((poses, foc, pp), 1), HW, K0inv)
    if sc.tied_focal:
        J[:, :, 8] = J[:, :, 7]
    return J


C_Q = 8.0


def _quat_unprojected(sc: Scene64, q):
    """(m, 9, 4): dR/dq with the normalisation's projection left out (R of q / |q0| for a fixed |q0|), and q / |q0|.
    quat_backward forms this gradient first and projects it after, so its rounding scales with these magnitudes."""
    nrm = q.norm(dim=-1, keepdim=True)

    def f(x, n):
        x, y, z, w = (x / n).unbind(-1)
        return torch.stack((1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                            2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                            2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)))
    return torch.func.vmap(torch.func.jacfwd(f))(q, nrm).abs(), (q / nrm).abs()


def _quat_term(Hraw9, Ju, qh):
    """C_Q u (|g_u,theta| + |qhat_theta| sum_j |g_u,j|), g_u = the unprojected quaternion gradient's magnitude."""
    gu = torch.einsum('mk,mkj->mj', Hraw9, Ju)
    return C_Q * U * (gu + qh * gu.sum(-1, keepdim=True))


def small_bound(sc: Scene64, T):
    """(bound, fixed-point part of it) for every element of the small gradient, in the `small` layout."""
    o = sc.offsets()
    n, E = sc.n, sc.E
    Hent, Hent_fix, Hraw = [], [], []
    Himg = torch.zeros((n, 12), dtype=F64)
    Himg_fix = torch.zeros((n, 12), dtype=F64)
    Himg_raw = torch.zeros((n, 9), dtype=F64)
    for k, p in enumerate(T['per']):
        Ga, qa, w, kap = p['G'].abs(), p['q'].abs(), p['w'].abs(), p['kappa']
        GQ = (Ga[:, :, None] * qa[:, None, :]).sum(0).reshape(-1)          # sum |G_a| |q_b|
        KQ = ((w * kap)[:, None] * qa).sum(0).repeat(3)                     # sum w kappa |q_b|, every a
        h = torch.cat((GQ, Ga.sum(0)))
        hk = torch.cat((KQ, (w * kap).sum().repeat(3)))
        c = 2 * sc.chain_ent[k] * U + EPS_RSQRT
        Hent.append(c * h + hk)
        Hraw.append(h)
        Hent_fix.append(torch.full((12,), sc.n_partials_ent[k] * FIX_Q, dtype=F64))
        g = T['geo'][p['i']]
        wk = (w * kap + C3 * U * p['Gn'])[:, None]
        ci = 2 * sc.chain_img[p['i']] * U + EPS_RSQRT
        GC = 2 * (Ga * g['Cn'][:, None]).sum(0)                              # sum |G_a| |C|, every b
        Himg[p['i'], :9] += (ci * GC + 2 * (wk * g['Cn'][:, None]).sum(0)).repeat_interleave(3)
        Himg[p['i'], 9:] += ci * Ga.sum(0) + (wk[:, 0]).sum()
        Himg_raw[p['i']] += GC.repeat_interleave(3)
    for i in range(n):
        Himg_fix[i] = sc.n_partials_img[i] * FIX_Q
    Je = _edge_jacobian(sc).abs()
    Ji = _image_jacobian(sc).abs()
    bound = torch.zeros(o['total'], dtype=F64)
    fixed = torch.zeros(o['total'], dtype=F64)
    edge_b = torch.zeros((E, 10), dtype=F64)
    edge_f = torch.zeros((E, 10), dtype=F64)
    edge_a = torch.zeros((E, 10), dtype=F64)
    for k in range(len(T['per'])):
        e = int(sc.ent_edge[k])
        edge_b[e] += Hent[k] @ Je[e]
        edge_f[e] += Hent_fix[k] @ Je[e]
        edge_a[e] += Hraw[k] @ Je[e]
    if sc.norm_pw_scale:               # the mean over every edge's log-scale gradient: their errors, its fp32 block sum, -
        kc = math.ceil(E / 256) + 13
        a_mean = edge_a[:, 7].sum() / E
        edge_b[:, 7] += edge_b[:, 7].sum() / E + (kc + 2) * U * a_mean + U * edge_a[:, 7]
        edge_f[:, 7] += edge_f[:, 7].sum() / E
    edge_b = edge_b + edge_f
    # rounding inside quat_backward: before the projection onto the tangent of |q| = 1
    o_ = sc.offsets()
    Ju, qh = _quat_unprojected(sc, sc.small[o_['pw']:o_['adapt']].reshape(E, 8)[:, :4])
    edge_raw9 = torch.zeros((E, 9), dtype=F64)
    for k in range(len(T['per'])):
        edge_raw9[int(sc.ent_edge[k])] += Hraw[k][:9]
    edge_b[:, :4] += _quat_term(edge_raw9, Ju, qh) * _edge_scale(sc)[:, None]
    Ju, qh = _quat_unprojected(sc, sc.small[o_['poses']:o_['focals']].reshape(n, 7)[:, :4])
    img_q = _quat_term(Himg_raw, Ju, qh)
    img_b = torch.einsum('nk,nkt->nt', Himg + Himg_fix, Ji)
    img_b[:, :4] += img_q
    img_f = torch.einsum('nk,nkt->nt', Himg_fix, Ji)
    for b, src_e, src_i in ((bound, edge_b, img_b), (fixed, edge_f, img_f)):
        b[o['poses']:o['focals']] = src_i[:, :7].reshape(-1)
        b[o['focals']:o['pp']] = src_i[:, 7:9].reshape(-1)
        b[o['pp']:o['pw']] = src_i[:, 9:11].reshape(-1)
        b[o['pw']:o['adapt']] = src_e[:, :8].reshape(-1)
        b[o['adapt']:] = src_e[:, 8:].reshape(-1)
    return bound, fixed


def _edge_scale(sc: Scene64):
    """max_b s adapt_b of every edge: M = s R diag(adapt), so dL/dR = dL/dM s adapt."""
    M, _ = edge_transforms(sc, sc.small)
    return M.norm(dim=1).max(-1).values


# ---------------------------------------------------------------------------------------------- the Adam step
EPS_APPROX = 2.0 ** -22       # sqrt.approx.f32 / rcp.approx.f32: PTX documents 2^-23 relative and 1 ulp; twice that


def adam64(p, m, v, g, step_size, bc2s, approx, dg=0.0, beta1=0.9, beta2=0.9, eps=1e-8):
    """One torch.optim.Adam step (base_opt.py's betas) in float64 from fp32 state p, m, v, gradient g and the fp32
    schedule row (step_size = lr / (1 - beta1^t), bc2s = sqrt(1 - beta2^t)), with the fp32 constants the kernels use
    (beta = fl32(0.9), 1 - beta exact).  Returns (p, m, v) after the step and a bound of each for the kernel's fp32
    arithmetic: every operation rounds once (u), sqrt and 1/x are MUFU approximations (EPS_APPROX) on the streaming
    kernel's per-pixel path (`approx`), IEEE elsewhere; dg bounds the error of g itself.
      m' = b1 m + (1-b1) g                |dm'| <= 4u ((1-b1)(|g| + |m|) + b1 |m|) + (1-b1) dg
      v' = b2 v + (1-b2) g^2              |dv'| <= 4u (b2 v + (1-b2) g^2) + (1-b2)(2 |g| dg + dg^2)
      D  = sqrt(v')/bc2s + eps            |dD|  <= (dv' / (2 sqrt v') or sqrt dv', + e_sqrt sqrt v') / bc2s + 3u D
      p' = p - step m' / D                |dp'| <= step (|dm'| / D + |m'| |dD| / D^2) + |step m'/D| (e_rcp + 3u) + u |p'|"""
    f32 = lambda x: float(np.float32(x))
    b1, b2, eps = f32(beta1), f32(beta2), f32(eps)
    c1, c2 = 1.0 - b1, 1.0 - b2
    m1 = b1 * m + c1 * g
    v1 = b2 * v + c2 * g * g
    sv = v1.sqrt()
    den = sv / bc2s + eps
    upd = step_size * m1 / den
    p1 = p - upd
    e_op = EPS_APPROX if approx else U
    em = 4 * U * (c1 * (g.abs() + m.abs()) + b1 * m.abs()) + c1 * dg
    ev = 4 * U * (b2 * v.abs() + c2 * g * g) + c2 * (2 * g.abs() * dg + dg * dg)
    dsv = torch.where(v1 > 0, ev / (2 * torch.where(v1 > 0, sv, torch.ones_like(sv))), ev.sqrt()) + e_op * sv
    dden = dsv / bc2s + 3 * U * den
    eupd = step_size * (em / den + m1.abs() * dden / den.square()) + upd.abs() * (e_op + 3 * U)
    return p1, m1, v1, eupd + U * p1.abs(), em, ev


# ---------------------------------------------------------------------------------------------- mutations (resolution)
def ratio(err, bound):
    """max err / bound over the elements (0 / 0 counts as 0)."""
    err, bound = torch.as_tensor(err, dtype=F64), torch.as_tensor(bound, dtype=F64)
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    return float(r.max()) if r.numel() else 0.0


def wrap_pixels(sc: Scene64, img):
    """Pixels B of pixel pairs (2j, 2j+1) of the streaming layout whose row wraps inside the pair (u_B == 0): the
    `uB == W` branch of unproject_slots.  Pairs are counted from the image's first pixel, as the slots are."""
    H, W = sc.imshapes[img]
    pB = np.arange(1, H * W, 2)
    return pB[pB % W == 0]


def mutate_column(sc: Scene64, T, img, p):
    """Per-pixel gradient of image `img` with pixel p unprojected one column to the right (u + 1): the change at p."""
    g = T['geo'][img]
    dcol = g['d'][p] / (sc.small[sc.offsets()['focals'] + 2 * img] / sc.focal_break).exp()
    Y2 = g['Y'][p] + dcol * g['R'][:, 0]
    X2 = Y2 + g['T']
    new = 0.0
    for k, pk in enumerate(T['per']):
        if pk['i'] != img:
            continue
        e = pk['e']
        r = X2 - (pk['q'][p] @ T['M'][e].T + T['t'][e])
        w = pk['w'][p]
        G = w * r / r.norm() if sc.dist == 'l1' else 2 * w * r
        new = new + float((G * Y2).sum())
    return new - float(T['gd'][img][p])


def drop_entry_pixel(T, k, p):
    """Change of the per-pixel gradient when entry k's contribution to pixel p is dropped."""
    return -float(T['per'][k]['contrib'][p])


def resolution_demo(sc: Scene64, T, sbound, g_small_ref, img=0, n_cand=64):
    """The three mutations of a kernel the bound must be able to see, each built on the float64 side.  For every one:
    (caught, missed) = (perturbation / bound at the affected element, perturbation / (1e-4 max |ref|) of the affected
    tensor): caught > 1 means the element-wise bound sees it, missed <= 1 means the per-tensor criterion of the existing
    gradient tests does not.  Of the candidates the one the tensor criterion is least likely to see is reported."""
    out = {}
    gd_all = torch.cat(T['gd'])
    gmax = float(gd_all.abs().max())
    # 1. one pixel's u moved by one column at a row wrap inside a pixel pair
    best = None
    for i, (H, W) in enumerate(sc.imshapes):
        if W % 2 == 0:
            continue
        for p in wrap_pixels(sc, i)[:n_cand]:
            d = abs(mutate_column(sc, T, i, int(p)))
            cand = (d / float(T['gd_bound'][i][p]), d / (1e-4 * gmax))
            if cand[0] > 1 and (best is None or cand[1] < best[1]):
                best = cand
    out['column_at_pair_wrap'] = best
    # 2. one entry's contribution to one pixel dropped: the pixel with the smallest nonzero gradient of image `img`
    g0 = T['gd'][img].abs()
    p = int(torch.where(g0 > 0, g0, torch.full_like(g0, math.inf)).argmin())
    best = None
    for k, pk in enumerate(T['per']):
        if pk['i'] != img or pk['contrib'][p] == 0:
            continue
        d = abs(drop_entry_pixel(T, k, p))
        cand = (d / float(T['gd_bound'][img][p]), d / (1e-4 * gmax))
        if best is None or (cand[0] > 1, -cand[1]) > (best[0] > 1, -best[1]):
            best = cand
    out['entry_dropped_at_pixel'] = best
    # 3. one pixel's contribution missing from one entry's sums
    o = sc.offsets()
    ref_pw = g_small_ref[o['pw']:o['adapt']].abs().max()
    ref_ad = g_small_ref[o['adapt']:].abs().max()
    Je = _edge_jacobian(sc)
    best = None
    for k, pk in enumerate(T['per'][:8]):
        e = pk['e']
        h = torch.cat(((pk['G'][:, :, None] * pk['q'][:, None, :]).reshape(-1, 9), pk['G']), 1)
        dg = h @ Je[e]                                                   # (P, 10)
        b = torch.cat((sbound[o['pw'] + 8 * e:o['pw'] + 8 * e + 8], sbound[o['adapt'] + 2 * e:o['adapt'] + 2 * e + 2]))
        caught = (dg.abs() / b).max(1).values
        missed = torch.maximum(dg[:, :8].abs().max(1).values / (1e-4 * ref_pw), dg[:, 8:].abs().max(1).values / (1e-4 * ref_ad))
        ok = caught > 1
        if ok.any():
            j = int(torch.where(ok, missed, torch.full_like(missed, math.inf)).argmin())
            cand = (float(caught[j]), float(missed[j]))
            if best is None or cand[1] < best[1]:
                best = cand
    out['pixel_missing_from_entry_sums'] = best
    return out
