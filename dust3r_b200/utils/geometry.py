"""Small geometry helpers used by the host side of the two hot paths (API mirror of the subset of
dust3r/utils/geometry.py the paths touch: xy_grid :15-37, geotrf :40-101, inv :104-111,
depthmap_to_pts3d :114-162, depthmap_to_absolute_camera_coordinates :165-225)."""
from __future__ import annotations

import numpy as np
import torch


def xy_grid(W, H, device=None, origin=(0, 0), unsqueeze=None, cat_dim=-1, homogeneous=False, **arange_kw):
    """(H,W,2) grid with out[j,i] = (i + origin[0], j + origin[1]); numpy when device is None."""
    if device is None:
        xs = np.arange(origin[0], origin[0] + W, **arange_kw)
        ys = np.arange(origin[1], origin[1] + H, **arange_kw)
        grid = tuple(np.meshgrid(xs, ys, indexing='xy'))
        if homogeneous:
            grid = grid + (np.ones((H, W)),)
        if unsqueeze is not None:
            grid = tuple(np.expand_dims(g, unsqueeze) for g in grid[:2])
        return np.stack(grid, cat_dim) if cat_dim is not None else grid
    xs = torch.arange(origin[0], origin[0] + W, device=device, **arange_kw)
    ys = torch.arange(origin[1], origin[1] + H, device=device, **arange_kw)
    grid = tuple(torch.meshgrid(xs, ys, indexing='xy'))
    if homogeneous:
        grid = grid + (torch.ones((H, W), device=device),)
    if unsqueeze is not None:
        grid = (grid[0].unsqueeze(unsqueeze), grid[1].unsqueeze(unsqueeze))
    return torch.stack(grid, cat_dim) if cat_dim is not None else grid


def geotrf(Trf, pts, ncol=None, norm=False):
    """Apply a (batched) linear / affine / projective transform to points with last dim 2 or 3."""
    assert Trf.ndim >= 2
    if isinstance(Trf, np.ndarray):
        pts = np.asarray(pts)
    else:
        pts = torch.as_tensor(pts, dtype=Trf.dtype)
    out_shape = pts.shape[:-1]
    ncol = ncol or pts.shape[-1]
    d = pts.shape[-1]
    if Trf.ndim >= 3:
        nb = Trf.ndim - 2
        assert Trf.shape[:nb] == pts.shape[:nb], 'batch size does not match'
        Trf = Trf.reshape(-1, Trf.shape[-2], Trf.shape[-1])
        pts = pts.reshape(Trf.shape[0], -1, d) if pts.ndim > 2 else pts[:, None, :]
    else:
        pts = pts.reshape(-1, d)
    Tt = Trf.swapaxes(-1, -2)
    if d + 1 == Trf.shape[-1]:
        res = pts @ Tt[..., :-1, :] + Tt[..., -1:, :]
    elif d == Trf.shape[-1]:
        res = pts @ Tt
    else:
        raise ValueError(f'bad shapes {Trf.shape} x {pts.shape}')
    if norm:
        res = res / res[..., -1:]
        if norm != 1:
            res = res * norm
    return res[..., :ncol].reshape(*out_shape, ncol)


def inv(mat):
    if isinstance(mat, torch.Tensor):
        return torch.linalg.inv(mat)
    if isinstance(mat, np.ndarray):
        return np.linalg.inv(mat)
    raise ValueError(f'bad matrix type = {type(mat)}')


def depthmap_to_pts3d(depth, pseudo_focal, pp=None, **_):
    """depth (B,H,W), pseudo_focal (B,H,W) | (B,1,H,W) | (B,2,H,W) -> (B,H,W,3) camera-frame points."""
    B, H, W = depth.shape
    if pseudo_focal.ndim == 3:
        fx = fy = pseudo_focal
    elif pseudo_focal.ndim == 4:
        fx = pseudo_focal[:, 0]
        fy = pseudo_focal[:, 1] if pseudo_focal.shape[1] == 2 else fx
    else:
        raise NotImplementedError("Error, unknown input focal shape format.")
    assert fx.shape == depth.shape and fy.shape == depth.shape
    gx, gy = xy_grid(W, H, cat_dim=0, device=depth.device)[:, None]
    if pp is None:
        gx = gx - (W - 1) / 2
        gy = gy - (H - 1) / 2
    else:
        gx = gx.expand(B, -1, -1) - pp[:, 0, None, None]
        gy = gy.expand(B, -1, -1) - pp[:, 1, None, None]
    return torch.stack((depth * gx / fx, depth * gy / fy, depth), dim=-1)


def depthmap_to_camera_coordinates(depthmap, camera_intrinsics, pseudo_focal=None):
    camera_intrinsics = np.float32(camera_intrinsics)
    H, W = depthmap.shape
    assert camera_intrinsics[0, 1] == 0.0 and camera_intrinsics[1, 0] == 0.0
    if pseudo_focal is None:
        fu, fv = camera_intrinsics[0, 0], camera_intrinsics[1, 1]
    else:
        assert pseudo_focal.shape == (H, W)
        fu = fv = pseudo_focal
    cu, cv = camera_intrinsics[0, 2], camera_intrinsics[1, 2]
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    z = depthmap
    X_cam = np.stack(((u - cu) * z / fu, (v - cv) * z / fv, z), axis=-1).astype(np.float32)
    return X_cam, depthmap > 0.0


def depthmap_to_absolute_camera_coordinates(depthmap, camera_intrinsics, camera_pose, **kw):
    X_cam, valid = depthmap_to_camera_coordinates(depthmap, camera_intrinsics)
    X_world = X_cam
    if camera_pose is not None:
        R, t = camera_pose[:3, :3], camera_pose[:3, 3]
        X_world = np.einsum("ik, vuk -> vui", R, X_cam) + t[None, None, :]
    return X_world, valid


def find_reciprocal_matches(P1, P2):
    """dust3r/utils/geometry.py:345-361: (reciprocal_in_P2 bool[len(P2)], nn2_in_P1 int[len(P2)], number of matches).
    P2[k] is a reciprocal match when the nearest point of P1 to it, nn2_in_P1[k], has P2[k] as ITS nearest point in P2.
    CUDA tensors (N,3) / (M,3) are matched by a brute-force kernel on the GPU (csrc/scene_ops.cu) and returned as tensors;
    arrays / CPU tensors use scipy's cKDTree exactly like the reference and return numpy."""
    if torch.is_tensor(P1) and P1.is_cuda:
        from ..cloud_opt.scene_ops import nearest_neighbours
        P2 = torch.as_tensor(P2, device=P1.device)
        nn1_in_P2 = nearest_neighbours(P1, P2)
        nn2_in_P1 = nearest_neighbours(P2, P1)
        reciprocal_in_P2 = nn1_in_P2[nn2_in_P1] == torch.arange(len(nn2_in_P1), device=P1.device)
        return reciprocal_in_P2, nn2_in_P1, int(reciprocal_in_P2.sum())
    from scipy.spatial import cKDTree

    def nearest(src, dst):
        return cKDTree(dst).query(src, workers=8)[1]
    P1, P2 = np.asarray(P1), np.asarray(P2)
    to_p2, to_p1 = nearest(P1, P2), nearest(P2, P1)
    mutual_2 = to_p2[to_p1] == np.arange(len(to_p1))
    assert (to_p1[to_p2] == np.arange(len(to_p2))).sum() == mutual_2.sum()     # the relation is symmetric
    return mutual_2, to_p1, mutual_2.sum()


NORM_MODES = ('avg_dis',)
_REFERENCE_NORM_MODES = ('avg_log1p', 'avg_warp-log1p', 'median_dis', 'sqrt_dis')


def check_norm_mode(norm_mode):
    """A falsy mode (no normalisation) or one of NORM_MODES; the reference's other modes raise NotImplementedError."""
    if not norm_mode or norm_mode in NORM_MODES:
        return
    known = norm_mode in _REFERENCE_NORM_MODES
    raise (NotImplementedError if known else ValueError)(
        f'norm_mode={norm_mode!r} is {"not supported" if known else "unknown"}: supported modes are {NORM_MODES} or a falsy value')


def normalize_pointcloud(pts1, pts2, norm_mode='avg_dis', valid1=None, valid2=None, ret_factor=False):
    """dust3r/utils/geometry.py:249-308 for norm_mode 'avg_dis': both pointmaps (B,H,W,3) divided by the mean distance to the
    origin of the valid points of the two together (per batch item, clipped below at 1e-8).  Invalid points do not enter the
    mean, whatever they hold."""
    from .misc import invalid_to_zeros
    check_norm_mode(norm_mode)
    assert pts1.ndim >= 3 and pts1.shape[-1] == 3
    assert pts2 is None or (pts2.ndim >= 3 and pts2.shape[-1] == 3)
    z1, nnz1 = invalid_to_zeros(pts1, valid1, ndim=3)
    z2, nnz2 = invalid_to_zeros(pts2, valid2, ndim=3) if pts2 is not None else (None, 0)
    allp = torch.cat((z1, z2), dim=1) if pts2 is not None else z1
    factor = allp.norm(dim=-1).sum(dim=1) / (nnz1 + nnz2 + 1e-8)
    factor = factor.clip(min=1e-8)
    while factor.ndim < pts1.ndim:
        factor = factor.unsqueeze(-1)
    res = pts1 / factor
    if pts2 is not None:
        res = (res, pts2 / factor)
    if ret_factor:
        res = res + (factor,)
    return res


@torch.no_grad()
def get_joint_pointcloud_depth(z1, z2, valid_mask1, valid_mask2=None, quantile=0.5):
    """dust3r/utils/geometry.py:311-324: per batch item, the median (torch.nanmedian: the lower one) of the valid depths of
    both maps together; NaN for an item without any."""
    from .misc import invalid_to_nans
    zz = invalid_to_nans(z1, valid_mask1).reshape(len(z1), -1)
    if z2 is not None:
        zz = torch.cat((zz, invalid_to_nans(z2, valid_mask2).reshape(len(z2), -1)), dim=-1)
    if quantile == 0.5:
        return torch.nanmedian(zz, dim=-1).values
    return torch.nanquantile(zz, quantile, dim=-1)


@torch.no_grad()
def get_joint_pointcloud_center_scale(pts1, pts2, valid_mask1=None, valid_mask2=None, z_only=False, center=True):
    """dust3r/utils/geometry.py:327-342: per batch item, the per-coordinate median of the valid points of both maps (B,1,1,3)
    and the median distance of those points to it (B,1,1,1)."""
    from .misc import invalid_to_nans
    pp = invalid_to_nans(pts1, valid_mask1).reshape(len(pts1), -1, 3)
    if pts2 is not None:
        pp = torch.cat((pp, invalid_to_nans(pts2, valid_mask2).reshape(len(pts2), -1, 3)), dim=1)
    c = torch.nanmedian(pp, dim=1, keepdim=True).values
    if z_only:
        c[..., :2] = 0
    scale = torch.nanmedian(((pp - c) if center else pp).norm(dim=-1), dim=1).values
    return c[:, None, :, :], scale[:, None, None, None]
