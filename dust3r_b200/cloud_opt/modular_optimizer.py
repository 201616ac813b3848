"""ModularPointCloudOptimizer — per-image parameters so individual poses / intrinsics can be frozen
(API mirror of dust3r/cloud_opt/modular_optimizer.py).  Same fused CUDA step as PointCloudOptimizer;
the per-image `requires_grad` flags become the kernel's trainable mask, and the objective uses the
base-class normalisation (per-edge pixel means / n_edges, base_opt.py:246-273)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from .base_opt import BasePCOptimizer
from ..utils.geometry import geotrf, depthmap_to_pts3d
from ..utils.device import to_cpu, to_numpy


class ModularPointCloudOptimizer(BasePCOptimizer):
    def __init__(self, *args, optimize_pp=False, fx_and_fy=False, focal_brake=20, **kwargs):
        super().__init__(*args, **kwargs)
        self.has_im_poses = True
        self.focal_brake = focal_brake
        self.im_depthmaps = nn.ParameterList(torch.randn(H, W) / 10 - 3 for H, W in self.imshapes)
        self.im_poses = nn.ParameterList(self.rand_pose(self.POSE_DIM) for _ in range(self.n_imgs))
        default_focals = [self.focal_brake * np.log(max(H, W)) for H, W in self.imshapes]
        self.im_focals = nn.ParameterList(torch.FloatTensor([f, f] if fx_and_fy else [f]) for f in default_focals)
        self.im_pp = nn.ParameterList(torch.zeros((2,)) for _ in range(self.n_imgs))
        self.im_pp.requires_grad_(optimize_pp)

    def _engine_push(self, eng):
        dev = self.device
        logd = torch.cat([d.data.reshape(-1) for d in self.im_depthmaps]).contiguous()
        eng.set_params(logd, torch.stack([p.data for p in self.im_poses]),
                       torch.stack([f.data for f in self.im_focals]), torch.stack([p.data for p in self.im_pp]),
                       self.pw_poses.data, self.pw_adaptors.data,
                       train_poses=[p.requires_grad for p in self.im_poses],
                       train_focals=[p.requires_grad for p in self.im_focals],
                       train_pp=[p.requires_grad for p in self.im_pp],
                       train_pw=self.pw_poses.requires_grad, train_adaptors=self.pw_adaptors.requires_grad,
                       norm_pw_scale=self.norm_pw_scale)

        def pull():
            s = eng.get_small()
            off = 0
            for i, (H, W) in enumerate(self.imshapes):
                self.im_depthmaps[i].data.copy_(logd[off:off + H * W].view(H, W))
                off += H * W
                self.im_poses[i].data.copy_(s['im_poses'][i])
                self.im_focals[i].data.copy_(s['im_focals'][i])
                self.im_pp[i].data.copy_(s['im_pp'][i])
            self.pw_poses.data.copy_(s['pw_poses'])
            self.pw_adaptors.data.copy_(s['pw_adaptors'])
        return pull

    def _engine_params(self):
        return [*self.im_depthmaps, *self.im_poses, *self.im_focals, *self.im_pp, self.pw_poses, self.pw_adaptors]

    def _engine_grads(self, eng, logd_grad, small_grad):
        g = eng.split_small(small_grad)
        depth, off = [], 0
        for H, W in self.imshapes:
            depth.append(logd_grad[off:off + H * W].view(H, W))
            off += H * W
        return [*depth, *g['im_poses'].unbind(0), *g['im_focals'].unbind(0), *g['im_pp'].unbind(0), g['pw_poses'],
                g['pw_adaptors']]

    # ---------------------------------------------------------------- fixing parameters to known values
    # A preset writes the value into the per-image parameter and switches its gradient off; the fused step receives the
    # flags as its trainable mask (see _engine_push), so a preset image keeps exactly the value given here.
    def _select(self, msk):
        """Image indices addressed by `msk`: None = all, an int, a list / array / tensor of ints, or a boolean mask."""
        if msk is None:
            return list(range(self.n_imgs))
        if isinstance(msk, (int, np.integer)):
            return [int(msk)]
        arr = msk.detach().cpu().numpy() if torch.is_tensor(msk) else np.asarray(msk)
        if arr.dtype == np.bool_:
            assert len(arr) == self.n_imgs
            return np.flatnonzero(arr).tolist()
        if np.issubdtype(arr.dtype, np.integer):
            return arr.reshape(-1).tolist()
        raise ValueError(f'bad {msk=}')

    _get_msk_indices = _select   # reference name

    def _preset(self, what, setter, values, msk):
        for idx, value in zip(self._select(msk), values):
            if self.verbose:
                shown = value[:3, 3] if what == 'pose' else value
                print(f' (setting {what} #{idx} = {shown})')
            setter(idx, value).requires_grad_(False)

    def preset_pose(self, known_poses, pose_msk=None):
        if torch.is_tensor(known_poses) and known_poses.ndim == 2:
            known_poses = [known_poses]
        self._preset('pose', lambda i, pose: self._set_pose(self.im_poses, i, torch.as_tensor(pose), force=True), known_poses,
                     pose_msk)
        # with two or more cameras pinned the global scale is no longer a free gauge: stop normalising pairwise scales
        frozen = sum(1 for prm in self.im_poses if not prm.requires_grad)
        self.norm_pw_scale = frozen <= 1

    def preset_focal(self, known_focals, msk=None):
        self._preset('focal', lambda i, f: self._set_focal(i, f, force=True), known_focals, msk)

    def preset_principal_point(self, known_pp, msk=None):
        self._preset('principal point', lambda i, pp: self._set_principal_point(i, pp, force=True), known_pp, msk)

    def preset_intrinsics(self, known_intrinsics, msk=None):
        if torch.is_tensor(known_intrinsics) and known_intrinsics.ndim == 2:
            known_intrinsics = [known_intrinsics]
        assert all(tuple(K.shape) == (3, 3) for K in known_intrinsics)
        self.preset_focal([K.diagonal()[:2].mean() for K in known_intrinsics], msk)
        self.preset_principal_point([K[:2, 2] for K in known_intrinsics], msk)

    # ---------------------------------------------------------------- parameterisation
    # focal = exp(param / focal_brake) (one or two entries per image), principal point = image centre + 10 * param,
    # depth = exp(param); a setter only writes when the parameter is trainable or `force` is given.
    @staticmethod
    def _writable(param, force):
        return force or param.requires_grad

    def _set_focal(self, idx, focal, force=False):
        param = self.im_focals[idx]
        if self._writable(param, force):
            param.data.fill_(self.focal_brake * np.log(float(focal)))
        return param

    def _set_principal_point(self, idx, pp, force=False):
        param = self.im_pp[idx]
        if self._writable(param, force):
            H, W = self.imshapes[idx]
            centre = torch.tensor((W / 2, H / 2), dtype=param.dtype)
            param.data.copy_((torch.as_tensor(to_numpy(pp), dtype=param.dtype).cpu() - centre) / 10)
        return param

    def _set_depthmap(self, idx, depth, force=False):
        param = self.im_depthmaps[idx]
        if self._writable(param, force):
            param.data.copy_(depth.log().nan_to_num(neginf=0))
        return param

    def get_focals(self):
        return torch.exp(torch.stack(tuple(self.im_focals)) / self.focal_brake)

    def get_known_focal_mask(self):
        return torch.tensor([not prm.requires_grad for prm in self.im_focals])

    def get_principal_points(self):
        centres = torch.tensor([(W / 2, H / 2) for H, W in self.imshapes], dtype=self.im_pp[0].dtype, device=self.im_pp[0].device)
        return centres + 10 * torch.stack(tuple(self.im_pp))

    def get_intrinsics(self):
        f = self.get_focals().view(self.n_imgs, -1)     # (n, 1) shared focal or (n, 2) = (fx, fy)
        K = torch.zeros((self.n_imgs, 3, 3), device=self.device)
        K[:, 0, 0], K[:, 1, 1], K[:, 2, 2] = f[:, 0], f[:, -1], 1
        K[:, :2, 2] = self.get_principal_points()
        return K

    def get_im_poses(self):
        return self._get_poses(torch.stack(tuple(self.im_poses)))

    def get_depthmaps(self):
        return [logd.exp() for logd in self.im_depthmaps]

    def depth_to_pts3d(self):
        """World pointmaps of all images: from the fused step's own unprojection on CUDA, in torch otherwise."""
        if self.device.type == 'cuda':
            eng = self._get_engine()
            self._engine_push(eng)
            flat, out, off = eng.pts3d(), [], 0
            for H, W in self.imshapes:
                out.append(flat[off:off + H * W].view(H, W, 3))
                off += H * W
            return out
        focals, pps, poses, depths = self.get_focals(), self.get_principal_points(), self.get_im_poses(), self.get_depthmaps()
        out = []
        for i, (H, W) in enumerate(self.imshapes):
            f_map = focals[i][..., None, None].expand(1, *focals[i].shape, H, W)
            cam = depthmap_to_pts3d(depths[i][None], f_map, pp=pps[i:i + 1])[0]
            out.append(geotrf(poses[i], cam))
        return out

    def get_pts3d(self):
        return self.depth_to_pts3d()
