"""ORACLE (test infrastructure, not product code): CPU fp32 restatement of DUSt3R's global-alignment
loop (cloud_opt).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this file.

Parity status: pinned against the reference's own code executed here, with one caveat: the reference
needs `roma`, which is absent, so the pinning runs are "reference cloud_opt + local roma restatement"
(oracle/roma_stub; the stub's three entry points are themselves pinned against scipy's Rotation / weighted Kabsch
and a float64 closed-form Umeyama in tests/test_roma_stub.py).  tests/test_oracle_vs_reference.py re-checks it whenever /root/reference is mounted;
tests/golden/align_*.npz store the reference's loss trajectories and final parameters.

Restates (autograd does the backward, torch.optim.Adam the update, exactly as the reference):
  parameters / buffers ........ dust3r/cloud_opt/optimizer.py:22-61, base_opt.py:44-105
  pairwise poses + scale ...... base_opt.py:150-195 (quaternion XYZW normalised; T = signed_expm1;
                                rows 0..2 scaled by exp(s_e) * exp(log(base_scale) - mean(s)))
  adaptors .................... base_opt.py:143-148
  unprojection ................ optimizer.py:170-211 (PointCloudOptimizer),
                                modular_optimizer.py:118-142 + utils/geometry.py:114-162 (Modular)
  objective ................... optimizer.py:188-201 (stacked), base_opt.py:246-273 (per-edge mean)
  distances / conf transform .. commons.py:48-80
  loop, schedules, Adam ....... base_opt.py:326-366, commons.py:83-90, optim_factory.py:9-14
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Tuple

import numpy as np
import torch


def signed_expm1(x):
    return torch.sign(x) * torch.expm1(torch.abs(x))


def quat_xyzw_to_rotmat(q):
    q = q / q.norm(dim=-1, keepdim=True)
    x, y, z, w = q.unbind(-1)
    R = torch.stack((1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)), dim=-1)
    return R.reshape(q.shape[:-1] + (3, 3))


def conf_trf(conf, mode):
    if mode == 'log':
        return conf.log()
    if mode == 'sqrt':
        return conf.sqrt()
    if mode == 'm1':
        return conf - 1
    if mode in ('id', 'none'):
        return conf
    raise ValueError(mode)


def cosine_schedule(t, lr_start, lr_end):
    return lr_end + (lr_start - lr_end) * (1 + np.cos(t * np.pi)) / 2


def linear_schedule(t, lr_start, lr_end):
    return lr_start + (lr_end - lr_start) * t


@dataclass
class AlignProblem:
    """Observations of one scene: E directed edges over n images (flat pixel order = row-major)."""
    edges: List[Tuple[int, int]]
    imshapes: List[Tuple[int, int]]            # (H, W) per image
    pred_i: List[torch.Tensor]                 # E x (P_i, 3)
    pred_j: List[torch.Tensor]                 # E x (P_j, 3)
    weight_i: List[torch.Tensor]               # E x (P_i,)   already conf-transformed
    weight_j: List[torch.Tensor]
    dist: str = 'l1'
    base_scale: float = 0.5
    pw_break: float = 20.0
    focal_break: float = 20.0
    norm_pw_scale: bool = True
    variant: str = 'stacked'                   # 'stacked' = PointCloudOptimizer, 'per_edge' = Modular/base

    @property
    def n_imgs(self):
        return len(self.imshapes)

    @staticmethod
    def from_output(out, dist='l1', conf='log', variant='stacked', **kw):
        idx1 = [int(i) for i in out['view1']['idx']]
        idx2 = [int(j) for j in out['view2']['idx']]
        edges = list(zip(idx1, idx2))
        n = max(max(e) for e in edges) + 1
        p1, p2 = out['pred1']['pts3d'], out['pred2']['pts3d_in_other_view']
        c1, c2 = out['pred1']['conf'], out['pred2']['conf']
        imshapes = [None] * n
        for e, (i, j) in enumerate(edges):
            imshapes[i] = tuple(p1[e].shape[:2])
            imshapes[j] = tuple(p2[e].shape[:2])
        return AlignProblem(edges=edges, imshapes=imshapes,
                            pred_i=[p1[e].reshape(-1, 3).float() for e in range(len(edges))],
                            pred_j=[p2[e].reshape(-1, 3).float() for e in range(len(edges))],
                            weight_i=[conf_trf(c1[e].reshape(-1).float(), conf) for e in range(len(edges))],
                            weight_j=[conf_trf(c2[e].reshape(-1).float(), conf) for e in range(len(edges))],
                            dist=dist, variant=variant, **kw)


def init_params(prob: AlignProblem, seed=0, fx_and_fy=False):
    """Same distributions as the reference draws (optimizer.py:29-32, base_opt.py:90) from a seeded
    generator, so reference / oracle / CUDA can all start from identical values."""
    g = torch.Generator().manual_seed(seed)
    n, E = prob.n_imgs, len(prob.edges)
    P = dict()
    P['im_depthmaps'] = [torch.randn((H * W,), generator=g) / 10 - 3 for H, W in prob.imshapes]
    P['im_poses'] = torch.randn((n, 7), generator=g)
    f0 = torch.tensor([[prob.focal_break * math.log(max(H, W))] * (2 if fx_and_fy else 1) for H, W in prob.imshapes],
                      dtype=torch.float32)
    P['im_focals'] = f0
    P['im_pp'] = torch.zeros((n, 2))
    P['pw_poses'] = torch.randn((E, 8), generator=g)
    P['pw_adaptors'] = torch.zeros((E, 2))
    return P


def pw_transforms(prob, pw_poses, pw_adaptors):
    R = quat_xyzw_to_rotmat(pw_poses[:, :4])
    T = signed_expm1(pw_poses[:, 4:7])
    s = pw_poses[:, 7].exp()
    if prob.norm_pw_scale:
        s = s * (math.log(prob.base_scale) - pw_poses[:, 7].mean()).exp()
    adapt = torch.cat((pw_adaptors[:, 0:1], pw_adaptors), dim=-1)
    if prob.norm_pw_scale:
        adapt = adapt - adapt.mean(dim=1, keepdim=True)
    adapt = (adapt / prob.pw_break).exp()
    return s[:, None, None] * R, s[:, None] * T, adapt


def unproject(prob, im_depthmaps, im_poses, im_focals, im_pp):
    """-> list of (P_i, 3) world points."""
    R = quat_xyzw_to_rotmat(im_poses[:, :4])
    T = signed_expm1(im_poses[:, 4:7])
    f = (im_focals / prob.focal_break).exp()
    out = []
    for i, (H, W) in enumerate(prob.imshapes):
        d = im_depthmaps[i].exp()
        dt = d.dtype               # float32 for the oracle itself; float64 when the float64 tests evaluate it
        v, u = torch.meshgrid(torch.arange(H, dtype=dt), torch.arange(W, dtype=dt), indexing='ij')
        cx = W / 2 + 10 * im_pp[i, 0]
        cy = H / 2 + 10 * im_pp[i, 1]
        fx, fy = f[i, 0], f[i, -1]
        cam = torch.stack((d * (u.reshape(-1) - cx) / fx, d * (v.reshape(-1) - cy) / fy, d), dim=-1)
        out.append(cam @ R[i].T + T[i])
    return out


def _dist(a, b, w, kind):
    if kind == 'l1':
        return (a - b).norm(dim=-1) * w
    if kind == 'l2':
        return (a - b).square().sum(dim=-1) * w
    raise ValueError(kind)


def loss_fn(prob: AlignProblem, P):
    sR, sT, adapt = pw_transforms(prob, P['pw_poses'], P['pw_adaptors'])
    X = unproject(prob, P['im_depthmaps'], P['im_poses'], P['im_focals'], P['im_pp'])
    areas = [h * w for h, w in prob.imshapes]
    if prob.variant == 'stacked':
        tot_i = sum(areas[i] for i, j in prob.edges)
        tot_j = sum(areas[j] for i, j in prob.edges)
    li = lj = 0
    loss = 0
    for e, (i, j) in enumerate(prob.edges):
        ai = (adapt[e] * prob.pred_i[e]) @ sR[e].T + sT[e]
        aj = (adapt[e] * prob.pred_j[e]) @ sR[e].T + sT[e]
        di = _dist(X[i], ai, prob.weight_i[e], prob.dist)
        dj = _dist(X[j], aj, prob.weight_j[e], prob.dist)
        if prob.variant == 'stacked':
            li = li + di.sum()
            lj = lj + dj.sum()
        else:
            loss = loss + di.mean() + dj.mean()
    if prob.variant == 'stacked':
        return li / tot_i + lj / tot_j
    return loss / len(prob.edges)


def align_oracle(prob: AlignProblem, P0, niter=300, lr=0.01, schedule='cosine', lr_min=1e-6,
                 trainable=('im_depthmaps', 'im_poses', 'im_focals', 'pw_poses'), record_every=1):
    """Runs the reference loop (base_opt.py:326-366).  Returns (losses, final params)."""
    P = {}
    for k, v in P0.items():
        if isinstance(v, list):
            P[k] = [t.clone().float().requires_grad_(k in trainable) for t in v]
        else:
            P[k] = v.clone().float().requires_grad_(k in trainable)
    params = []
    for k in P:
        if k in trainable:
            params += P[k] if isinstance(P[k], list) else [P[k]]
    opt = torch.optim.Adam(params, lr=lr, betas=(0.9, 0.9))
    losses = []
    for it in range(niter):
        t = it / niter
        cur = cosine_schedule(t, lr, lr_min) if schedule == 'cosine' else linear_schedule(t, lr, lr_min)
        for gp in opt.param_groups:
            gp['lr'] = cur
        opt.zero_grad()
        loss = loss_fn(prob, P)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    final = {k: ([t.detach() for t in v] if isinstance(v, list) else v.detach()) for k, v in P.items()}
    return losses, final
