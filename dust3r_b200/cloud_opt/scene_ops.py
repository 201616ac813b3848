"""CUDA versions of the scene-level operators either side of the alignment loop (SURVEY §8f): thin host wrappers over
csrc/scene_ops.cu.  Each takes CUDA fp32 tensors on an H100 and mirrors the host port it accelerates:

  clean_pointcloud      cloud_opt/pointcloud_filter.py   (dust3r/cloud_opt/base_opt.py:369-405)
  rigid_registration    cloud_opt/commons.py             (roma.rigid_points_registration as used by init_im_poses.py)
  weiszfeld_focal       post_process.py                  (dust3r/post_process.py:12-60)
  nearest_neighbours    utils/geometry.py                (find_reciprocal_matches, dust3r/utils/geometry.py:345-361)
  segment_sky           viz.py                           (dust3r/viz.py:345-381, csrc/sky_ops.cu)

The host ports dispatch here when their inputs live on the GPU; CPU tensors keep the reference's own CPU algorithms (as the
reference does: these run once per scene, not per iteration)."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib


def _f32(t):
    return t.to(torch.float32).contiguous()


@torch.no_grad()
def clean_pointcloud(im_confs, K, cams, depthmaps, all_pts3d, tol=0.001, bad_conf=0):
    """Per-image lists (any mix of image sizes) -> list of new confidence maps, same shapes as im_confs."""
    dev = im_confs[0].device
    _lib.require_cuda_device(dev)
    n = len(im_confs)
    assert n == len(cams) == len(K) == len(depthmaps) == len(all_pts3d)
    assert 0 <= tol < 1
    shapes = [tuple(c.shape) for c in im_confs]
    areas = [h * w for h, w in shapes]
    off = np.zeros(n + 1, dtype=np.int64)
    off[1:] = np.cumsum(areas)
    conf = torch.cat([_f32(c).reshape(-1) for c in im_confs])
    pts = torch.cat([_f32(p).reshape(-1, 3) for p in all_pts3d])
    depth = torch.cat([_f32(d).reshape(-1) for d in depthmaps])
    Kd = _f32(torch.stack([torch.as_tensor(k) for k in K]).to(dev)).reshape(n, 9)
    Td = _f32(torch.stack([torch.as_tensor(c) for c in cams]).to(dev)).reshape(n, 16)
    hw = torch.tensor(shapes, dtype=torch.int32, device=dev)
    offd = torch.from_numpy(off).to(dev)
    _lib.launch(dev, 'd3r_clean_pointcloud', n, hw.data_ptr(), offd.data_ptr(), int(max(areas)), pts.data_ptr(), conf.data_ptr(),
                depth.data_ptr(), Kd.data_ptr(), Td.data_ptr(), float(tol), float(bad_conf))
    return [conf[off[i]:off[i + 1]].reshape(shapes[i]).to(im_confs[i].dtype) for i in range(n)]


@torch.no_grad()
def rigid_registration(x, y, weights, compute_scaling=True):
    """Weighted Umeyama / Kabsch for B problems at once: x, y (B,P,3) or (P,3), weights (B,P) or (P,) ->
    (R (B,3,3), t (B,3)[, s (B,)]) minimising sum w |s R x + t - y|^2.  The O(P) moments come from one kernel (fp64
    accumulation); the 3x3 SVDs run in fp64 on the device."""
    single = x.ndim == 2
    if single:
        x, y, weights = x[None], y[None], weights[None]
    dev = x.device
    _lib.require_cuda_device(dev)
    B, P = int(x.shape[0]), int(x.shape[1])
    x, y, w = _f32(x), _f32(y), _f32(weights)
    m = torch.empty((B, 17), dtype=torch.float64, device=dev)
    _lib.launch(dev, 'd3r_procrustes_moments', B, P, x.data_ptr(), y.data_ptr(), w.data_ptr(), m.data_ptr())
    sw = m[:, 0]
    xm, ym = m[:, 1:4] / sw[:, None], m[:, 4:7] / sw[:, None]
    M = m[:, 7:16].reshape(B, 3, 3) - sw[:, None, None] * ym[:, :, None] * xm[:, None, :]      # sum w (y - ym)(x - xm)^T
    varx = m[:, 16] - sw * (xm * xm).sum(dim=-1)                                                  # sum w |x - xm|^2
    U, S, Vh = torch.linalg.svd(M)
    d = torch.sign(torch.linalg.det(U @ Vh))
    D = torch.ones_like(S)
    D[:, -1] = d
    R = U @ torch.diag_embed(D) @ Vh
    if compute_scaling:
        s = (S * D).sum(dim=-1) / varx
        t = ym - s[:, None] * (R @ xm[:, :, None])[:, :, 0]
        out = (R.float(), t.float(), s.float())
    else:
        t = ym - (R @ xm[:, :, None])[:, :, 0]
        out = (R.float(), t.float())
    return tuple(o[0] for o in out) if single else out


@torch.no_grad()
def weiszfeld_focal(pts3d, pp, steps=10):
    """pts3d (B,H,W,3) camera-frame pointmaps, pp (B,2) -> (B,) focals (before the caller's clipping)."""
    dev = pts3d.device
    _lib.require_cuda_device(dev)
    B, H, W, _ = pts3d.shape
    p = _f32(pts3d)
    c = _f32(pp.to(dev)).reshape(B, 2)
    out = torch.empty((B,), dtype=torch.float32, device=dev)
    _lib.launch(dev, 'd3r_weiszfeld_focal', int(B), int(H), int(W), p.data_ptr(), c.data_ptr(), int(steps), out.data_ptr())
    return out


@torch.no_grad()
def nearest_neighbours(queries, points):
    """(N,3), (M,3) CUDA tensors -> (N,) int64 index of the nearest row of `points` for every query (squared Euclidean distance
    in fp32, the lowest index on exact ties).  Non-finite input: a point with a NaN coordinate is never chosen, and a query
    without any finite distance (a NaN query, or every point NaN) gets index 0."""
    dev = queries.device
    _lib.require_cuda_device(dev)
    q, p = _f32(queries).reshape(-1, 3), _f32(points.to(dev)).reshape(-1, 3)
    nn = torch.empty((q.shape[0],), dtype=torch.int32, device=dev)
    _lib.launch(dev, 'd3r_nearest_neighbours', int(q.shape[0]), int(p.shape[0]), q.data_ptr(), p.data_ptr(), nn.data_ptr())
    return nn.long()


def _quantise(x):
    """np.uint8(255 * x.clip(0, 1)) as numpy computes it (product in x's dtype, truncation toward zero); uint8 passes through."""
    return x if x.dtype == torch.uint8 else (255 * x.clamp(0, 1)).to(torch.uint8)


def _segment_sky_u8(rgb, shapes):
    """rgb: flat uint8 CUDA tensor holding the (H, W, 3) images of `shapes` back to back -> list of (H, W) bool masks."""
    dev = rgb.device
    _lib.require_cuda_device(dev)
    lib = _lib.get_lib()
    n = len(shapes)
    areas = [h * w for h, w in shapes]
    off = np.zeros(n + 1, dtype=np.int64)
    off[1:] = np.cumsum(areas)
    total = int(off[-1])
    assert rgb.numel() == 3 * total and rgb.dtype == torch.uint8
    hw = torch.tensor(shapes, dtype=torch.int32, device=dev)
    offd = torch.from_numpy(off[:n]).to(dev)
    out = torch.empty((total,), dtype=torch.uint8, device=dev)
    ws = torch.empty((int(lib.d3r_segment_sky_workspace_bytes(n, total)),), dtype=torch.uint8, device=dev)
    _lib.launch(dev, 'd3r_segment_sky', n, hw.data_ptr(), offd.data_ptr(), int(max(areas)), total, rgb.data_ptr(), out.data_ptr(),
                ws.data_ptr(), ws.numel())
    sky = out.view(torch.bool)
    return [sky[off[i]:off[i + 1]].view(shapes[i]) for i in range(n)]


@torch.no_grad()
def segment_sky(images):
    """List of (H, W, 3) RGB CUDA tensors (float in [0, 1] as scene.imgs holds them, or uint8; any mix of sizes) -> list of (H, W)
    bool sky masks on the device, one batched call (dust3r/viz.py:345-381, bit-exact)."""
    if not images:
        return []
    shapes = [tuple(x.shape[:2]) for x in images]
    assert all(x.ndim == 3 and x.shape[2] == 3 for x in images), 'segment_sky takes (H, W, 3) RGB images'
    rgb = torch.cat([_quantise(x).reshape(-1) for x in images])
    return _segment_sky_u8(rgb, shapes)


@torch.no_grad()
def segment_sky_host_images(images, device):
    """Like segment_sky for (H, W, 3) float32 numpy arrays in host memory (scene.imgs): the floats go up in one pinned copy and are
    quantised on the device."""
    if any(np.asarray(x).dtype != np.float32 for x in images):     # other dtypes are quantised in their own precision
        return segment_sky([torch.from_numpy(np.asarray(x)).to(device) for x in images])
    shapes = [tuple(x.shape[:2]) for x in images]
    assert all(x.ndim == 3 and x.shape[2] == 3 for x in images), 'segment_sky takes (H, W, 3) RGB images'
    total = 3 * sum(h * w for h, w in shapes)
    host = torch.empty((total,), dtype=torch.float32, pin_memory=True)
    np.concatenate([np.asarray(x, dtype=np.float32).reshape(-1) for x in images], out=host.numpy())
    return _segment_sky_u8(_quantise(host.to(device, non_blocking=True)), shapes)
