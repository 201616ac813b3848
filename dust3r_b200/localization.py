"""Visual localisation of a query image against map images of known geometry (dust3r_visloc/localization.py, visloc.py:80-172,
dust3r_visloc/evaluation.py), for one query at a time:

  run_pnp         the reference's PnP.  Numpy input runs its cv2.solvePnPRansac code unchanged; CUDA tensors run the loop on
                  the GPU (csrc/pnp_ops.cu: 5-point EPnP hypotheses, OpenCV's fp32 inlier test and stopping rule, the samples
                  from a counter-based generator instead of OpenCV's RNG) and then what OpenCV does after its loop:
                  cv2.solvePnP(SOLVEPNP_SQPNP) on the winning inliers as float64, on the host.
  pnp_ransac      the GPU loop alone: the winning hypothesis, its inliers and the number of hypotheses evaluated.
  localize        the body of visloc.py's loop for one query: one inference() call over every (query, map) pair, confidence
                  masks, reciprocal nearest neighbours, the matches mapped back to the query's original pixels and run_pnp,
                  all on the device up to the PnP refinement.
  get_pose_error, aggregate_stats   dust3r_visloc/evaluation.py (roma's geodesic distance restated: roma is not a dependency).
Only mode='cv2' exists: the reference's poselib and pycolmap modes need libraries this package does not use.
"""
from __future__ import annotations

import collections
import math
import random

import numpy as np
import torch

from . import _lib

CONFIDENCE = 0.9999
ITERATIONS = 10_000
DEFAULT_SEED = 0x5DEECE66D   # csrc/pnp_core.h kDefaultSeed: fixed, so results are deterministic


def _check_finite(pts2D, pts3D, K):
    for name, x in (('pts2D', pts2D), ('pts3D', pts3D), ('K', K)):
        ok = bool(torch.isfinite(x).all()) if torch.is_tensor(x) else bool(np.isfinite(np.asarray(x, np.float64)).all())
        if not ok:
            raise ValueError(f'run_pnp: {name} has non-finite values')


@torch.no_grad()
def pnp_ransac(pts2D, pts3D, K, reprojection_error=5.0, confidence=CONFIDENCE, max_iters=ITERATIONS, seed=DEFAULT_SEED):
    """PnP-RANSAC loop on the GPU for CUDA tensors pts2D (N,2) and pts3D (N,3), N >= 5, rounded to fp32 as OpenCV rounds them.
    Returns (result int32 (4,) = [best hypothesis or -1, its inlier count, hypotheses evaluated, 1], pose float64 (3,4) world ->
    camera [R | t] of the best hypothesis, inlier mask bool (N,)), all on the device, without synchronising."""
    dev = pts2D.device
    _lib.require_cuda_device(dev)
    p2 = pts2D.to(dev, torch.float32).reshape(-1, 2).contiguous()
    p3 = pts3D.to(dev, torch.float32).reshape(-1, 3).contiguous()
    if p2.shape[0] != p3.shape[0]:
        raise ValueError(f'pnp_ransac: {p2.shape[0]} 2-D points for {p3.shape[0]} 3-D points')
    K = np.asarray(K.cpu() if torch.is_tensor(K) else K, np.float64)
    n = p2.shape[0]
    ws = torch.empty((int(_lib.get_lib().d3r_pnp_ransac_workspace_bytes(int(max_iters))),), dtype=torch.uint8, device=dev)
    result = torch.empty((4,), dtype=torch.int32, device=dev)
    pose = torch.empty((12,), dtype=torch.float64, device=dev)
    mask = torch.empty((n,), dtype=torch.uint8, device=dev)
    _lib.launch(dev, 'd3r_pnp_ransac', int(n), p2.data_ptr(), p3.data_ptr(), float(K[0, 0]), float(K[1, 1]), float(K[0, 2]),
                float(K[1, 2]), float(reprojection_error), float(confidence), int(max_iters), int(seed), ws.data_ptr(), ws.numel(),
                result.data_ptr(), pose.data_ptr(), mask.data_ptr())
    R, t = pose[:9].reshape(3, 3), pose[9:]
    return result, torch.cat([R, t[:, None]], 1), mask.bool()


def _cv2_pose(success, r_pose, t_pose):
    import cv2
    if not success:
        return False, None
    r_pose = cv2.Rodrigues(r_pose)[0]                   # world2cam
    RT = np.r_[np.c_[r_pose, t_pose], [(0, 0, 0, 1)]]
    return True, np.linalg.inv(RT)                      # cam2world


def run_pnp(pts2D, pts3D, K, distortion=None, mode='cv2', reprojectionError=5, img_size=None):
    """dust3r_visloc/localization.py:30-52 -> (success, cam2world float64 4x4 or None).  `distortion`: OpenCV's model (the 2-D
    points are undistorted on the host first).  Numpy input runs cv2.solvePnPRansac(SOLVEPNP_SQPNP, 10 000 iterations,
    confidence 0.9999) as the reference does; CUDA tensors run the loop on the GPU (pnp_ransac) and refine the winning
    inliers with cv2.solvePnP(SOLVEPNP_SQPNP), which is what solvePnPRansac does after its loop.  Non-finite points or K
    raise ValueError."""
    if mode != 'cv2':
        raise ValueError(f"run_pnp: mode {mode!r} is not supported (only 'cv2')")
    import cv2
    if len(pts2D) <= 4:
        return False, None
    _check_finite(pts2D, pts3D, K)
    if not torch.is_tensor(pts2D):
        try:
            if distortion is not None:
                pts2D = cv2.undistortPoints(np.copy(pts2D), K, np.array(distortion), R=None, P=K).reshape((-1, 2))
            return _cv2_pose(*cv2.solvePnPRansac(pts3D, pts2D, K, None, flags=cv2.SOLVEPNP_SQPNP, iterationsCount=ITERATIONS,
                                                 reprojectionError=reprojectionError, confidence=CONFIDENCE)[:3])
        except Exception as e:   # the reference reports and fails
            print(f'error during pnp: {e}')
            return False, None
    K = np.asarray(K.cpu() if torch.is_tensor(K) else K, np.float64)
    dev = pts2D.device
    if distortion is not None:
        und = cv2.undistortPoints(pts2D.detach().cpu().numpy(), K, np.array(distortion), R=None, P=K).reshape((-1, 2))
        pts2D = torch.from_numpy(np.ascontiguousarray(und)).to(dev)
    p2 = pts2D.to(dev, torch.float32).reshape(-1, 2).contiguous()
    p3 = pts3D.to(dev, torch.float32).reshape(-1, 3).contiguous()
    result, _, mask = pnp_ransac(p2, p3, K, reprojectionError)
    if int(result[0]) < 0:
        return False, None
    keep = mask.nonzero().squeeze(1)
    obj = p3[keep].double().cpu().numpy()
    img = p2[keep].double().cpu().numpy()
    try:
        ok, rvec, tvec = cv2.solvePnP(obj, img, K, None, flags=cv2.SOLVEPNP_SQPNP)
    except cv2.error as e:
        print(f'error during pnp: {e}')
        return False, None
    return _cv2_pose(ok, rvec, tvec)


def _flat_xy(mask):
    """xy_grid(W, H)[mask] of the reference, as int64 (K, 2) on the device: the (x, y) of the set pixels in row-major order."""
    yx = mask.nonzero()
    return yx.flip(1)


def localize_matches(query_view, map_views, model, device, conf_thr=3.0):
    """visloc.py:80-165 for one query: the 2-D (query, original pixels, float64 (K, 2)) / 3-D (map geometry, (K, 3))
    correspondences of every map view, concatenated in map order, on the device.  One inference() call covers every pair."""
    from .inference import inference
    from .utils.geometry import find_reciprocal_matches, geotrf
    dev = torch.device(device)

    def view(img, idx):
        return dict(img=img.unsqueeze(0), true_shape=np.int32([img.shape[1:]]), idx=idx, instance=str(idx))
    q = view(query_view['rgb_rescaled'], 0)
    pairs = [(q, view(m['rgb_rescaled'], 1 + i)) for i, m in enumerate(map_views)]
    out = inference(pairs, model, dev, batch_size=len(pairs), verbose=False, keep_on_device=True, return_images=False)
    pred1, pred2 = out['pred1'], out['pred2']
    to_orig = torch.as_tensor(np.asarray(query_view['to_orig'], np.float64), device=dev)
    pts2d_all, pts3d_all = [], []
    for i, map_view in enumerate(map_views):
        valid_map = torch.as_tensor(map_view['valid_rescaled'], device=dev)
        # pair i of a stacked batch, or of the per-pair lists inference() returns for mixed sizes
        c1, c2 = pred1['conf'][i], pred2['conf'][i]
        c1, c2 = c1.reshape(c1.shape[-2:]), c2.reshape(c2.shape[-2:])
        masks = [c1 >= conf_thr, (c2 >= conf_thr) & valid_map]
        pts3d = [pred1['pts3d'][i].reshape(c1.shape + (3,)), pred2['pts3d_in_other_view'][i].reshape(c2.shape + (3,))]
        xy = [_flat_xy(m) for m in masks]
        PQ, PM = pts3d[0][masks[0]], pts3d[1][masks[1]]
        if len(PQ) == 0 or len(PM) == 0:
            continue
        reciprocal_in_PM, nnM_in_PQ, _ = find_reciprocal_matches(PQ, PM)
        matches_im1 = xy[1][reciprocal_in_PM]
        matches_im0 = xy[0][nnM_in_PQ][reciprocal_in_PM]
        if len(matches_im1) == 0:
            continue
        map_pts3d = torch.as_tensor(map_view['pts3d_rescaled'], device=dev)
        pts3d_all.append(map_pts3d[matches_im1[:, 1], matches_im1[:, 0]])
        pts2d_all.append(geotrf(to_orig, matches_im0.double() + 0.5, norm=True) - 0.5)   # cv2 -> colmap, rescale, -> cv2
    if not pts2d_all:
        return None, None
    return torch.cat(pts2d_all), torch.cat(pts3d_all)


def localize(query_view, map_views, model, device, conf_thr=3.0, reprojection_error=5.0, reprojection_error_diag_ratio=None,
             pnp_max_points=100_000, rng=random):
    """visloc.py:80-172 for one query view against its map views (the reference's view-dict keys: rgb_rescaled, to_orig,
    intrinsics, distortion, rgb; map views also valid_rescaled and pts3d_rescaled) -> (success, cam2world float64 4x4 or
    None).  At most pnp_max_points correspondences go to the PnP, chosen by rng.sample on the host as the reference does."""
    pts2d, pts3d = localize_matches(query_view, map_views, model, device, conf_thr)
    if pts2d is None:
        return False, None
    pts2d = pts2d.float()
    if len(pts2d) > pnp_max_points:
        idxs = torch.as_tensor(rng.sample(range(len(pts2d)), pnp_max_points), device=pts2d.device)
        pts3d, pts2d = pts3d[idxs], pts2d[idxs]
    W, H = query_view['rgb'].size
    thr = reprojection_error if reprojection_error_diag_ratio is None else reprojection_error_diag_ratio * math.sqrt(W ** 2 + H ** 2)
    return run_pnp(pts2d, pts3d, query_view['intrinsics'], query_view['distortion'], 'cv2', thr, img_size=[W, H])


def get_pose_error(pr_camtoworld, gt_cam_to_world):
    """dust3r_visloc/evaluation.py:get_pose_error -> (translation error, rotation error in degrees) as float64 tensors.  The
    angle is roma.rotmat_geodesic_distance, restated: 2 asin(|R2 - R1|_F / (2 sqrt 2)), from |R2 - R1|_F = 2 sqrt 2 sin(a / 2)."""
    pr, gt = torch.as_tensor(np.asarray(pr_camtoworld)), torch.as_tensor(np.asarray(gt_cam_to_world))
    abs_transl_error = torch.linalg.norm(pr[:3, 3] - gt[:3, 3])
    d = torch.linalg.norm(gt[:3, :3] - pr[:3, :3], dim=(-1, -2)) / (2.0 * np.sqrt(2))
    return abs_transl_error, 2.0 * torch.asin(torch.clamp(d, -1.0, 1.0)) * 180 / np.pi


def aggregate_stats(info_str, pose_errors, angular_errors):
    """dust3r_visloc/evaluation.py:aggregate_stats: the median errors and the accuracy at the four (m, deg) thresholds."""
    stats = collections.Counter()
    median_pos_error = np.median(pose_errors)
    median_angular_error = np.median(angular_errors)
    out_str = f'{info_str}: {len(pose_errors)} images - {median_pos_error=}, {median_angular_error=}'
    for trl_thr, ang_thr in [(0.1, 1), (0.25, 2), (0.5, 5), (5, 10)]:
        for pose_error, angular_error in zip(pose_errors, angular_errors):
            stats[trl_thr, ang_thr] += (pose_error < trl_thr) and (angular_error < ang_thr)
    stats = {f'acc@{key[0]:g}m,{key[1]}deg': 100 * val / len(pose_errors) for key, val in stats.items()}
    for metric, perf in stats.items():
        out_str += f'  - {metric:12s}={float(perf):.3f}'
    return out_str
