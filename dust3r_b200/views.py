"""The view stage of evaluation datasets: RGB-D frames -> the view dicts `loss_of_one_batch` consumes, bit-identical to what
the reference's BaseStereoViewDataset.__getitem__ returns (dust3r/datasets/base/base_stereo_view_dataset.py
`_crop_resize_if_necessary` with dust3r/datasets/utils/cropping.py, ImgNorm, depthmap_to_absolute_camera_coordinates,
transpose_to_landscape).  Dataset-specific work -- which frames make an item, reading their files -- stays with the caller
(INTEGRATION.md); what is shared by every dataset happens here:

    frame = dict(img=uint8 (H, W, 3) RGB, depthmap=fp32 (H, W), camera_intrinsics=fp32 3x3, [camera_pose=fp32 4x4 cam2world],
                 [dataset=..., label=..., instance=...])
    views = prepare_views([frame1, frame2], (512, 384), rng=item_rng(seed, idx), idx=idx)
    view1, view2 = prepare_batch([(idx, [frame1, frame2]), ...], (512, 384), seed=seed)

The host plan (`plan_view`) restates the reference's crop / rescale / intrinsics arithmetic with its dtypes (fp32 intrinsics
updated by fp64 operands, rounded once per update) and its random draws; the pixel work of every view of a call runs in one
C-ABI call, `d3r_prepare_views` (csrc/view_ops.cu).  device='cpu' runs the same plan through Pillow, OpenCV and numpy, the
reference's own CPU algorithm.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

PASS_THROUGH = ('dataset', 'label', 'instance')


def item_rng(seed, idx):
    """The Generator BaseStereoViewDataset.__getitem__ uses for item `idx` of a dataset built with a (non-zero) `seed`."""
    return np.random.default_rng(seed=seed + idx)


def _resolution(resolution):
    """int or (width, height) with width >= height, as BaseStereoViewDataset accepts one resolution."""
    w, h = (resolution, resolution) if isinstance(resolution, (int, np.integer)) else tuple(resolution)
    if not all(isinstance(s, (int, np.integer)) and s > 0 for s in (w, h)) or w < h:
        raise ValueError(f'resolution must be a positive int or (width, height) ints with width >= height, got {resolution!r}')
    return int(w), int(h)


def _host_array(x):
    return x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def _check_frame(frame, i):
    """Shape, dtype and finiteness checks of one frame -> (H, W, intrinsics, pose or None) as numpy arrays.  The depth values
    are checked later, on the pixels the view samples (_check_depth)."""
    img = frame['img']
    if tuple(img.shape[2:]) != (3,) or len(img.shape) != 3 or img.dtype not in (np.uint8, torch.uint8):
        raise ValueError(f'frame {i}: img must be uint8 (H, W, 3) RGB, got {img.dtype} {tuple(img.shape)}')
    H, W = int(img.shape[0]), int(img.shape[1])
    depth = frame['depthmap']
    if tuple(depth.shape) != (H, W) or depth.dtype not in (np.float32, torch.float32):
        raise ValueError(f'frame {i}: depthmap must be float32 {(H, W)}, got {depth.dtype} {tuple(depth.shape)}')
    K = _host_array(frame['camera_intrinsics'])
    if K.shape != (3, 3) or K.dtype != np.float32:
        raise ValueError(f'frame {i}: camera_intrinsics must be a float32 3x3 array, got {K.dtype} {K.shape}')
    if not np.isfinite(K).all():
        raise ValueError(f'frame {i}: non-finite camera_intrinsics')
    if K[0, 1] != 0 or K[1, 0] != 0:
        raise ValueError(f'frame {i}: skewed camera_intrinsics (K[0, 1] = {K[0, 1]}, K[1, 0] = {K[1, 0]})')
    pose = frame.get('camera_pose')
    if pose is not None:
        pose = _host_array(pose)
        if pose.shape != (4, 4) or pose.dtype != np.float32:
            raise ValueError(f'frame {i}: camera_pose must be a float32 4x4 array, got {pose.dtype} {pose.shape}')
        if not np.isfinite(pose).all():
            raise ValueError(f'frame {i}: non-finite camera_pose')
    return H, W, K, pose


def _r32(x):
    """A float64 value rounded once to fp32: numpy's in-place update of an fp32 array by an fp64 (or int64) operand."""
    return np.float32(np.float64(x))


def _colmap_shift(K, offset, scaling=None):
    """cropping.camera_matrix_of_crop's update of an fp32 matrix: +0.5 on the principal point, the first two rows times
    `scaling` (fp64), the principal point minus `offset` (fp64), -0.5."""
    K = K.copy()
    for i in range(2):
        K[i, 2] = _r32(np.float64(K[i, 2]) + 0.5)
    if scaling is not None:
        for i in range(2):
            for j in range(3):
                K[i, j] = _r32(np.float64(K[i, j]) * scaling)
    for i in range(2):
        K[i, 2] = _r32(np.float64(K[i, 2]) - offset[i])
        K[i, 2] = _r32(np.float64(K[i, 2]) - 0.5)
    return K


def final_crop_box(K, centred, resolution, size1):
    """cropping.bbox_from_intrinsics_in_out: the box that moves the fp32 principal point of K to that of `centred`, rounded
    half to even.  Raises ValueError when it leaves the resized image of size1 = (W1, H1), where the reference would cut a
    depth map of the wrong shape."""
    l2, t2 = (int(v) for v in np.int32(np.round(K[:2, 2] - centred[:2, 2])))
    box = (l2, t2, l2 + resolution[0], t2 + resolution[1])
    if l2 < 0 or t2 < 0 or box[2] > size1[0] or box[3] > size1[1]:
        raise ValueError(f'final crop box {box} leaves the resized {size1[0]}x{size1[1]} image')
    return box


def plan_view(hw, intrinsics, resolution, rng, aug_crop=False):
    """Everything `_crop_resize_if_necessary` decides for a frame of hw = (H, W) pixels with fp32 `intrinsics`, drawing from
    `rng` exactly as it does.  Returns dict(crop1 = the principal-point crop box (l, t, r, b), portrait, resolution = (width,
    height) after the orientation choice, scale (fp64 scale_final), size1 = (W1, H1) of the resized crop, method ('lanczos' /
    'bicubic'), crop2 = the final crop box in the resized crop, intrinsics = the final fp32 3x3 before any transpose)."""
    from .utils.image import _BICUBIC, _LANCZOS
    H, W = hw
    cx, cy = (int(c) for c in np.round(intrinsics[:2, 2]))
    mx, my = min(cx, W - cx), min(cy, H - cy)
    if mx <= 0 or my <= 0:
        raise ValueError(f'principal point ({cx}, {cy}) leaves no crop inside the {W}x{H} frame')
    crop1 = (cx - mx, cy - my, cx + mx, cy + my)
    K = intrinsics.copy()
    K[0, 2] = _r32(np.float64(K[0, 2]) - crop1[0])
    K[1, 2] = _r32(np.float64(K[1, 2]) - crop1[1])
    Wc, Hc = 2 * mx, 2 * my

    w, h = resolution
    portrait = False
    if Hc > 1.1 * Wc:
        portrait = True
    elif 0.9 < Hc / Wc < 1.1 and w != h:
        portrait = bool(rng.integers(2))
    res = (h, w) if portrait else (w, h)
    grow = int(rng.integers(0, aug_crop)) if aug_crop > 1 else 0

    scale = max((res[0] + grow) / Wc, (res[1] + grow) / Hc) + 1e-8
    W1, H1 = int(np.floor(Wc * scale)), int(np.floor(Hc * scale))
    method = _LANCZOS if scale < 1 else _BICUBIC
    K = _colmap_shift(K, (0.5 * (Wc * scale - W1), 0.5 * (Hc * scale - H1)), scaling=scale)

    if W1 < res[0] or H1 < res[1]:
        raise ValueError(f'resized crop {W1}x{H1} is smaller than the resolution {res[0]}x{res[1]}')
    crop2 = final_crop_box(K, _colmap_shift(K, (0.5 * (W1 - res[0]), 0.5 * (H1 - res[1]))), res, (W1, H1))
    l2, t2 = crop2[:2]
    K[0, 2] = _r32(np.float64(K[0, 2]) - l2)
    K[1, 2] = _r32(np.float64(K[1, 2]) - t2)
    return dict(crop1=crop1, portrait=portrait, resolution=res, scale=scale, size1=(W1, H1), method=method, crop2=crop2,
                intrinsics=K)


def _plan_item(frames, resolution, rng, aug_crop):
    """Plans of the views of one item in order, then the 'rng' tag of each: the draws of __getitem__."""
    if rng is None:
        raise ValueError('a numpy Generator is required (rng=..., or seed=... for prepare_batch)')
    checked = [_check_frame(f, i) for i, f in enumerate(frames)]
    plans = [plan_view((H, W), K, resolution, rng, aug_crop) for H, W, K, _ in checked]
    tags = [int.from_bytes(rng.bytes(4), 'big') for _ in frames]
    return [dict(p, pose=pose, rng=tag) for p, (_, _, _, pose), tag in zip(plans, checked, tags)]


def _transposed(plan):
    """transpose_to_landscape stores a view whose width is below its height transposed."""
    w, h = plan['resolution']
    return w < h


def _out_shapes(plan):
    w, h = plan['resolution']
    return (w, h) if _transposed(plan) else (h, w)


def _view_host(frame, plan):
    """The reference's CPU algorithm on one frame: Pillow crop + resize + crop, ImgNorm, OpenCV nearest resize of the depth,
    numpy unprojection -> (img (3, h, w), depthmap, pts3d, valid_mask) as stored after transpose_to_landscape."""
    import PIL.Image
    import cv2
    from .utils.image import _LANCZOS, norm_lut
    l, t, r, b = plan['crop1']
    l2, t2, r2, b2 = plan['crop2']
    method = PIL.Image.Resampling.LANCZOS if plan['method'] == _LANCZOS else PIL.Image.Resampling.BICUBIC
    pil = PIL.Image.fromarray(_host_array(frame['img'])).crop((l, t, r, b)).resize(plan['size1'], method)
    pixels = torch.from_numpy(np.array(pil.crop((l2, t2, r2, b2)), dtype=np.uint8)).long()
    img = norm_lut()[pixels].permute(2, 0, 1)
    depth = cv2.resize(np.ascontiguousarray(_host_array(frame['depthmap'])[t:b, l:r]), plan['size1'],
                       interpolation=cv2.INTER_NEAREST)[t2:b2, l2:r2]
    K = plan['intrinsics']
    h, w = depth.shape
    z = depth.astype(np.float64)
    x = ((np.arange(w, dtype=np.float64)[None, :] - np.float64(K[0, 2])) * z / np.float64(K[0, 0])).astype(np.float32)
    y = ((np.arange(h, dtype=np.float64)[:, None] - np.float64(K[1, 2])) * z / np.float64(K[1, 1])).astype(np.float32)
    pose = plan['pose'] if plan['pose'] is not None else np.full((4, 4), np.nan, dtype=np.float32)
    pts = np.stack([((pose[i, 0] * x + pose[i, 1] * y) + pose[i, 2] * depth) + pose[i, 3] for i in range(3)], axis=-1)
    valid = (depth > 0) & np.isfinite(pts).all(axis=-1)
    if _transposed(plan):
        img, depth, pts, valid = img.transpose(1, 2), depth.T, pts.transpose(1, 0, 2), valid.T
    return dict(img=img.contiguous(), depthmap=torch.from_numpy(np.ascontiguousarray(depth)),
                pts3d=torch.from_numpy(np.ascontiguousarray(pts)), valid_mask=torch.from_numpy(np.ascontiguousarray(valid)))


def _check_depth(named):
    """__getitem__'s assertion on the views' depth maps, (name, depth map) pairs -- the frame's depth at the pixels the crop
    and the nearest-neighbour resize sample, not the whole frame: ValueError naming the first view with a non-finite value.
    One device synchronise for all views of a call."""
    if not bool(torch.stack([torch.isfinite(d).all() for _, d in named]).all()):
        bad = next(name for name, d in named if not bool(torch.isfinite(d).all()))
        raise ValueError(f'{bad}: non-finite depth at pixels the view samples')


def view_descriptors(frames, plans, outs, dev):
    """The d3r_view_desc array of one d3r_prepare_views call for the (frame, plan) pairs, writing into the (img, depthmap,
    pts3d, valid_mask) tensors of `outs` (contiguous, on `dev`) -> (descriptors, every other tensor they point into: hold
    them until the call is queued).  Frames already on `dev` are read in place.  With dev = cpu the pointers are host pointers (tests/native/view_host.cpp)."""
    from . import _lib
    from .utils.image import _device_table, resample_table
    descs = (_lib.ViewDesc * len(frames))()
    keep = []
    tmp_bytes = []
    for d, frame, plan in zip(descs, frames, plans):
        src = torch.as_tensor(frame['img']).to(dev).contiguous()
        depth = torch.as_tensor(frame['depthmap']).to(dev).contiguous()
        keep += [src, depth]
        l, t, r, b = plan['crop1']
        W1, H1 = plan['size1']
        l2, t2, r2, b2 = plan['crop2']
        ybounds = resample_table(b - t, H1, plan['method'])[0][t2:b2]
        d.row0 = int(ybounds[:, 0].min())
        d.rows = int((ybounds[:, 0] + ybounds[:, 1]).max()) - d.row0
        W = int(src.shape[1])
        d.src, d.depth = src.data_ptr() + 3 * (t * W + l), depth.data_ptr() + 4 * (t * W + l)
        d.src_pitch = d.depth_pitch = W
        d.H0, d.W0, d.H1, d.W1 = b - t, r - l, H1, W1
        d.crop_x0, d.crop_y0, d.H2, d.W2 = l2, t2, b2 - t2, r2 - l2
        d.transpose = int(_transposed(plan))
        xb, xk, _ = _device_table(dev, d.W0, W1, plan['method'])
        yb, yk, _ = _device_table(dev, d.H0, H1, plan['method'])
        keep += [xb, xk, yb, yk]       # the shared table cache may drop them before the launch
        d.xbounds, d.xcoefs, d.ybounds, d.ycoefs = xb.data_ptr(), xk.data_ptr(), yb.data_ptr(), yk.data_ptr()
        K = plan['intrinsics']
        d.fu, d.fv, d.cu, d.cv = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
        pose = plan['pose']
        d.pose[:] = [float('nan')] * 12 if pose is None else [float(v) for v in pose[:3].reshape(-1)]
        tmp_bytes.append(d.rows * d.W2 * 3)
    out_keys = ('img', 'depthmap', 'pts3d', 'valid_mask')
    tmp = torch.empty((sum(tmp_bytes),), dtype=torch.uint8, device=dev)
    offset = 0
    for d, out, n in zip(descs, outs, tmp_bytes):
        d.tmp = tmp.data_ptr() + offset
        offset += n
        d.img, d.depthmap, d.pts3d, d.valid = (out[k].data_ptr() for k in out_keys)
    return descs, keep + [tmp]


def _run_device(frames, plans, outs, dev):
    """One d3r_prepare_views call for every (frame, plan) pair (see view_descriptors)."""
    from . import _lib
    from .utils.image import device_lut
    descs, keep = view_descriptors(frames, plans, outs, dev)
    desc_dev = torch.empty((len(frames) * ctypes.sizeof(_lib.ViewDesc),), dtype=torch.uint8, device=dev)
    _lib.launch(dev, 'd3r_prepare_views', len(frames), descs, desc_dev.data_ptr(), device_lut(dev).data_ptr())
    stream = torch.cuda.current_stream(dev)
    for t in keep + [desc_dev]:          # freed before the kernels ran, their memory must not go to another stream
        if t.device.type == 'cuda':
            t.record_stream(stream)


def _empty_outputs(plan, dev, batch=None):
    h, w = _out_shapes(plan)
    lead = () if batch is None else (batch,)
    return dict(img=torch.empty(lead + (3, h, w), dtype=torch.float32, device=dev),
                depthmap=torch.empty(lead + (h, w), dtype=torch.float32, device=dev),
                pts3d=torch.empty(lead + (h, w, 3), dtype=torch.float32, device=dev),
                valid_mask=torch.empty(lead + (h, w), dtype=torch.bool, device=dev))


def _small_keys(frame, plan, idx, v, dev):
    """The per-view keys other than the four pixel arrays, as __getitem__ leaves them."""
    w, h = plan['resolution']
    K = plan['intrinsics'][[1, 0, 2]] if _transposed(plan) else plan['intrinsics']
    pose = plan['pose'] if plan['pose'] is not None else np.full((4, 4), np.nan, dtype=np.float32)
    view = dict(camera_intrinsics=torch.from_numpy(np.ascontiguousarray(K)).to(dev),
                camera_pose=torch.from_numpy(np.ascontiguousarray(pose)).to(dev))
    view.update({k: frame[k] for k in PASS_THROUGH if k in frame})
    view.update(idx=(idx[0], idx[1], v), true_shape=torch.tensor((h, w), dtype=torch.int32, device=dev), rng=plan['rng'])
    return view


def _device(device):
    dev = torch.device(device)
    if dev.type == 'cpu':
        return dev
    from . import _lib
    return _lib.cuda_device(dev)


def _item_idx(idx):
    return (int(idx[0]), int(idx[1])) if isinstance(idx, tuple) else (int(idx), 0)


@torch.no_grad()
def prepare_views(frames, resolution, *, rng, idx=0, aug_crop=False, device='cuda'):
    """The views BaseStereoViewDataset.__getitem__(idx) returns when its `_get_views` yields `frames` (see the module
    docstring for a frame) at `resolution` (int or (width, height), width >= height): one dict per frame with img (3, h, w)
    in [-1, 1], depthmap, camera_intrinsics, camera_pose (NaN without one), pts3d, valid_mask, true_shape, idx = (idx, ar_idx,
    view index), rng and the frame's dataset / label / instance; portrait views stored transposed as transpose_to_landscape
    leaves them.  `rng` is the item's numpy Generator (item_rng(seed, idx) for a seeded dataset); `idx` an int or the
    (idx, ar_idx) pair of an aspect-ratio sampler; aug_crop > 1 enlarges the resize target by rng.integers(0, aug_crop).
    Tensors are on `device`; on an H100 the pixel work of all frames is one d3r_prepare_views call, device='cpu' runs
    Pillow, OpenCV and numpy.  Raises ValueError on non-finite pose, skewed or non-fp32 intrinsics, crops that leave the
    frame, and (as the reference asserts on the view's depth map) non-finite depth at a pixel the view samples."""
    dev = _device(device)
    res = _resolution(resolution)
    plans = _plan_item(frames, res, rng, aug_crop)
    idx = _item_idx(idx)
    if dev.type == 'cpu':
        pixels = [_view_host(f, p) for f, p in zip(frames, plans)]
    else:
        pixels = [_empty_outputs(p, dev) for p in plans]
        _run_device(frames, plans, pixels, dev)
    _check_depth([(f'view {v}', px['depthmap']) for v, px in enumerate(pixels)])
    return [dict(_small_keys(f, p, idx, v, dev), **px) for v, (f, p, px) in enumerate(zip(frames, plans, pixels))]


@torch.no_grad()
def prepare_batch(items, resolution, *, seed=None, rng=None, aug_crop=False, device='cuda'):
    """A list of (idx, frames) items (two frames each) -> (view1, view2), what torch's default_collate makes of the
    reference dataset's items: pixel arrays, intrinsics, poses and true_shape stacked on `device`, idx a list of three int64
    tensors, rng an int64 tensor, dataset / label / instance lists.  With a non-zero `seed` each item draws from
    item_rng(seed, idx) as a seeded dataset reseeds per item; otherwise all items draw in order from `rng`.  On an H100 every
    view of the batch, of any mix of frame sizes and orientations, goes through one d3r_prepare_views call.  Feed the result
    to loss_of_one_batch(..., symmetrize_batch=True)."""
    from torch.utils.data import default_collate
    dev = _device(device)
    res = _resolution(resolution)
    items = list(items)
    if not items:
        raise ValueError('prepare_batch needs at least one item')
    plans, idxs = [], []
    for idx, frames in items:
        if len(frames) != 2:
            raise ValueError(f'item {idx!r} has {len(frames)} frames; a batch item is a pair of views')
        idxs.append(_item_idx(idx))
        plans.append(_plan_item(frames, res, item_rng(seed, idxs[-1][0]) if seed else rng, aug_crop))
    if len({_out_shapes(p) for pair in plans for p in pair}) != 1:
        raise ValueError('views of one batch must have the same landscape size')
    B = len(items)
    if dev.type == 'cpu':
        slots = []
        for v in range(2):
            per_item = [_view_host(items[b][1][v], plans[b][v]) for b in range(B)]
            slots.append({k: torch.stack([px[k] for px in per_item]) for k in per_item[0]})
    else:
        slots = [_empty_outputs(plans[0][v], dev, batch=B) for v in range(2)]
        order = [(b, v) for v in range(2) for b in range(B)]
        _run_device([items[b][1][v] for b, v in order], [plans[b][v] for b, v in order],
                    [{k: t[b] for k, t in slots[v].items()} for b, v in order], dev)
    _check_depth([(f'item {idxs[b][0]} view {v}', slots[v]['depthmap'][b]) for v in range(2) for b in range(B)])
    views = []
    for v in range(2):
        small = [_small_keys(items[b][1][v], plans[b][v], idxs[b], v, 'cpu') for b in range(B)]
        view = default_collate(small)
        for k in ('camera_intrinsics', 'camera_pose', 'true_shape'):
            view[k] = view[k].to(dev)
        view.update(slots[v])
        views.append(view)
    return tuple(views)
