"""PointCloudOptimizer — stacked-parameter global aligner (API mirror of
dust3r/cloud_opt/optimizer.py).  Parameters keep the reference's names, shapes and parametrisation
(log-depth padded to max_area, poses as XYZW quaternion + signed-log1p translation, focal as
focal_break*log f, principal point as offset/10) so state dicts interchange; the optimisation itself
runs in the fused CUDA step."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from .base_opt import BasePCOptimizer
from ..utils.geometry import xy_grid, geotrf
from ..utils.device import to_numpy


def _ravel_hw(tensor, fill=0):
    """(H, W, ...) -> (H*W, ...), zero-padded at the end up to `fill` rows (images of different sizes share one stack)."""
    flat = tensor.flatten(0, 1)
    missing = fill - flat.shape[0]
    if missing > 0:
        flat = torch.cat((flat, flat.new_zeros((missing,) + tuple(flat.shape[1:]))))
    return flat


def ParameterStack(params, keys=None, is_param=None, fill=0):
    """Stack per-image tensors (optionally picked from a dict by `keys`, optionally flattened + padded to `fill` pixels)
    into one float tensor; it becomes an nn.Parameter when the inputs were trainable or `is_param` is set."""
    items = list(params) if keys is None else [params[k] for k in keys]
    trainable = items[0].requires_grad
    assert all(it.requires_grad == trainable for it in items)
    if fill > 0:
        items = [_ravel_hw(it, fill) for it in items]
    stacked = torch.stack(items).float().detach()
    if is_param or trainable:
        stacked = nn.Parameter(stacked, requires_grad=trainable)
    return stacked


class PointCloudOptimizer(BasePCOptimizer):
    def __init__(self, *args, optimize_pp=False, focal_break=20, **kwargs):
        super().__init__(*args, **kwargs)
        self.has_im_poses = True
        self.focal_break = focal_break

        # same draws, same order as optimizer.py:29-33 so a shared torch seed gives a shared start
        depth0 = [torch.randn(H, W) / 10 - 3 for H, W in self.imshapes]
        poses0 = [self.rand_pose(self.POSE_DIM) for _ in range(self.n_imgs)]
        focals0 = [torch.FloatTensor([self.focal_break * np.log(max(H, W))]) for H, W in self.imshapes]
        pp0 = [torch.zeros((2,)) for _ in range(self.n_imgs)]

        self.imshape = self.imshapes[0]
        im_areas = [h * w for h, w in self.imshapes]
        self.max_area = max(im_areas)

        self.im_depthmaps = nn.Parameter(torch.stack([_ravel_hw(d, self.max_area) for d in depth0]).float())
        self.im_poses = nn.Parameter(torch.stack(poses0).float())
        self.im_focals = nn.Parameter(torch.stack(focals0).float())
        self.im_pp = nn.Parameter(torch.stack(pp0).float())
        self.im_pp.requires_grad_(optimize_pp)
        self.register_buffer('_pp', torch.tensor([(w / 2, h / 2) for h, w in self.imshapes]))
        self.register_buffer('_ei', torch.tensor([i for i, j in self.edges]))
        self.register_buffer('_ej', torch.tensor([j for i, j in self.edges]))
        self.total_area_i = sum(im_areas[i] for i, j in self.edges)
        self.total_area_j = sum(im_areas[j] for i, j in self.edges)

    # the reference also registers _grid/_weight_*/_stacked_pred_* buffers (optimizer.py:45-57); here
    # they exist only inside the engine's packed float4 observation buffer.

    def _engine_variant(self):
        return 'stacked'

    def _engine_pix_stride(self):
        return self.max_area

    def _engine_push(self, eng):
        eng.set_params(self.im_depthmaps.data.view(-1), self.im_poses.data, self.im_focals.data, self.im_pp.data,
                       self.pw_poses.data, self.pw_adaptors.data,
                       train_poses=self.im_poses.requires_grad, train_focals=self.im_focals.requires_grad,
                       train_pp=self.im_pp.requires_grad, train_pw=self.pw_poses.requires_grad,
                       train_adaptors=self.pw_adaptors.requires_grad, norm_pw_scale=self.norm_pw_scale)

        def pull():
            s = eng.get_small()
            self.im_poses.data.copy_(s['im_poses'])
            self.im_focals.data.copy_(s['im_focals'])
            self.im_pp.data.copy_(s['im_pp'])
            self.pw_poses.data.copy_(s['pw_poses'])
            self.pw_adaptors.data.copy_(s['pw_adaptors'])
        return pull

    # ---------------------------------------------------------------- fixing parameters to known values
    # The stacked optimizer keeps one tensor per parameter kind, so a preset must cover EVERY image and freezes the
    # whole kind (use ModularPointCloudOptimizer to pin a subset of the cameras).
    def _get_msk_indices(self, msk):
        """Image indices addressed by `msk`: None = all, an int, a list / array / tensor of ints, or a boolean mask."""
        if msk is None:
            return np.arange(self.n_imgs)
        if isinstance(msk, (int, np.integer)):
            return np.array([int(msk)])
        arr = msk.detach().cpu().numpy() if torch.is_tensor(msk) else np.asarray(msk)
        if arr.dtype == np.bool_:
            assert len(arr) == self.n_imgs
            return np.flatnonzero(arr)
        if np.issubdtype(arr.dtype, np.integer):
            return arr.reshape(-1)
        raise ValueError(f'bad {msk=}')

    def _preset_all(self, what, stacked_param, setter, values, msk):
        picked = self._get_msk_indices(msk)
        assert len(picked) == self.n_imgs and np.all(picked == np.arange(self.n_imgs)), 'incomplete mask!'
        assert stacked_param.requires_grad, 'it must be True at this point, otherwise no modification occurs'
        for idx, value in zip(picked, values):
            if self.verbose:
                shown = value[:3, 3] if what == 'pose' else value
                print(f' (setting {what} #{idx} = {shown})')
            setter(int(idx), value)
        stacked_param.requires_grad_(False)

    def preset_pose(self, known_poses, pose_msk=None):
        if torch.is_tensor(known_poses) and known_poses.ndim == 2:
            known_poses = [known_poses]
        self._preset_all('pose', self.im_poses, lambda i, pose: self._set_pose(self.im_poses, i, torch.as_tensor(pose)),
                         known_poses, pose_msk)
        self.norm_pw_scale = False      # all cameras pinned: the global scale is no longer a free gauge

    def preset_focal(self, known_focals, msk=None):
        self._preset_all('focal', self.im_focals, self._set_focal, known_focals, msk)

    def preset_principal_point(self, known_pp, msk=None):
        self._preset_all('principal point', self.im_pp, self._set_principal_point, known_pp, msk)

    # ---------------------------------------------------------------- parameterisation
    # focal = exp(im_focals / focal_break), principal point = image centre + 10 * im_pp, depth = exp(im_depthmaps);
    # setters write one image's row and only when the stack is trainable (or `force`).
    def _row(self, stacked_param, idx, force):
        row = stacked_param[idx]
        return row, (force or row.requires_grad)

    def _set_focal(self, idx, focal, force=False):
        row, writable = self._row(self.im_focals, idx, force)
        if writable:
            row.data.fill_(self.focal_break * np.log(float(focal)))
        return row

    def _set_principal_point(self, idx, pp, force=False):
        row, writable = self._row(self.im_pp, idx, force)
        if writable:
            offset = torch.as_tensor(to_numpy(pp), dtype=row.dtype).cpu() - self._pp[idx].cpu()
            row.data.copy_(offset / 10)
        return row

    def _set_depthmap(self, idx, depth, force=False):
        row, writable = self._row(self.im_depthmaps, idx, force)
        if writable:
            row.data.copy_(_ravel_hw(depth, self.max_area).log().nan_to_num(neginf=0))
        return row

    def get_focals(self):
        return torch.exp(self.im_focals / self.focal_break)

    def get_known_focal_mask(self):
        return torch.full((self.n_imgs,), not self.im_focals.requires_grad, dtype=torch.bool)

    def get_principal_points(self):
        return self._pp + 10 * self.im_pp

    def get_intrinsics(self):
        K = torch.zeros((self.n_imgs, 3, 3), device=self.device)
        K[:, 0, 0] = K[:, 1, 1] = self.get_focals().flatten()
        K[:, :2, 2] = self.get_principal_points()
        K[:, 2, 2] = 1
        return K

    def get_im_poses(self):
        return self._get_poses(self.im_poses)

    def get_depthmaps(self, raw=False):
        stack = self.im_depthmaps.exp()
        if raw:
            return stack
        return [row[:h * w].view(h, w) for row, (h, w) in zip(stack, self.imshapes)]

    def depth_to_pts3d(self):
        """(n, max_area, 3) world-frame pointmaps.  On the GPU this is one launch of the engine's
        unprojection kernel; before `.to(cuda)` it is evaluated with torch ops (host glue, not timed)."""
        if self.device.type == 'cuda':
            eng = self._get_engine()
            self._engine_push(eng)
            return eng.pts3d().view(self.n_imgs, self.max_area, 3)
        pixels = torch.stack([_ravel_hw(xy_grid(W, H, device=self.device).float(), self.max_area) for H, W in self.imshapes])
        depth = self.get_depthmaps(raw=True).unsqueeze(-1)
        centred = pixels - self.get_principal_points().unsqueeze(1)
        # (depth * centred) / focal, in this order: bit-identical to the reference's CPU evaluation
        cam = torch.cat((depth * centred / self.get_focals().unsqueeze(1), depth), dim=-1)
        return geotrf(self.get_im_poses(), cam)
