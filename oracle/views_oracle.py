"""CPU restatement of the reference's view stage (dust3r/datasets/base/base_stereo_view_dataset.py `_crop_resize_if_necessary`
and `__getitem__`, dust3r/datasets/utils/cropping.py, dust3r/utils/geometry.py depthmap_to_absolute_camera_coordinates,
transpose_to_landscape) with the libraries the reference uses: Pillow for the image, OpenCV for the depth map, numpy for the
intrinsics (fp32 arrays updated in place, so numpy's own type promotion decides every rounding) and the unprojection (einsum).
It follows the reference's control flow step by step and shares no code with dust3r_b200.views, whose plan it checks.

    views_oracle(frames, (512, 384), rng, idx=3, aug_crop=16) -> list of view dicts as __getitem__ returns them (numpy arrays,
    img a torch tensor, portrait views transposed).
"""
import hashlib

import numpy as np
import PIL.Image
import torch


def digest(x):
    """sha256 of an array's dtype, shape and bytes, NaNs made one bit pattern (tests/golden/views.npz stores view arrays so):
    equal digests = equal arrays, NaN-aware, whatever the NaN payloads the producing code left."""
    a = np.ascontiguousarray(x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x))
    if a.dtype.kind == 'f':
        a = np.where(np.isnan(a), np.array(np.nan, dtype=a.dtype), a)
    return hashlib.sha256(f'{a.dtype.str}{a.shape}'.encode() + a.tobytes()).hexdigest()


def _img_norm(pil):
    """torchvision ToTensor + Normalize((0.5,) * 3, (0.5,) * 3) on an RGB image, with torch CPU ops."""
    x = torch.from_numpy(np.array(pil, dtype=np.uint8)).permute(2, 0, 1).contiguous().to(torch.float32).div(255)
    return x.sub_(0.5).div_(0.5)


def _crop(pil, depth, K, box):
    l, t, r, b = box
    K = K.copy()
    K[0, 2] -= l
    K[1, 2] -= t
    return pil.crop((l, t, r, b)), depth[t:b, l:r], K


def _to_colmap_and_scale(K, input_res, output_res, scaling=1, offset_factor=0.5):
    margins = np.asarray(input_res) * scaling - output_res
    assert np.all(margins >= 0.0)
    offset = offset_factor * margins
    out = K.copy()
    out[0, 2] += 0.5
    out[1, 2] += 0.5
    out[:2, :] *= scaling
    out[:2, 2] -= offset
    out[0, 2] -= 0.5
    out[1, 2] -= 0.5
    return out


def _rescale(pil, depth, K, target):
    import cv2
    in_res = np.array(pil.size)
    target = np.array(target)
    scale = max(target / pil.size) + 1e-8
    out_res = np.floor(in_res * scale).astype(int)
    pil = pil.resize(tuple(out_res), resample=PIL.Image.Resampling.LANCZOS if scale < 1 else PIL.Image.Resampling.BICUBIC)
    depth = cv2.resize(depth, out_res, fx=scale, fy=scale, interpolation=cv2.INTER_NEAREST)
    return pil, depth, _to_colmap_and_scale(K, in_res, out_res, scaling=scale)


def crop_resize(img, depth, K, resolution, rng, aug_crop=False):
    """_crop_resize_if_necessary -> (PIL image, depth map, intrinsics)."""
    pil = PIL.Image.fromarray(img)
    W, H = pil.size
    cx, cy = K[:2, 2].round().astype(int)
    mx, my = min(cx, W - cx), min(cy, H - cy)
    pil, depth, K = _crop(pil, depth, K, (cx - mx, cy - my, cx + mx, cy + my))
    W, H = pil.size
    if H > 1.1 * W:
        resolution = resolution[::-1]
    elif 0.9 < H / W < 1.1 and resolution[0] != resolution[1]:
        if rng.integers(2):
            resolution = resolution[::-1]
    target = np.array(resolution)
    if aug_crop > 1:
        target += rng.integers(0, aug_crop)
    pil, depth, K = _rescale(pil, depth, K, target)
    K2 = _to_colmap_and_scale(K, pil.size, resolution, offset_factor=0.5)
    l, t = np.int32(np.round(K[:2, 2] - K2[:2, 2]))
    return _crop(pil, depth, K, (l, t, l + resolution[0], t + resolution[1]))


def unproject(depth, K, pose):
    """depthmap_to_absolute_camera_coordinates + the finiteness mask of __getitem__ -> (pts3d, valid_mask)."""
    K = np.float32(K)
    fu, fv, cu, cv = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    u, v = np.meshgrid(np.arange(depth.shape[1]), np.arange(depth.shape[0]))
    X = np.stack(((u - cu) * depth / fu, (v - cv) * depth / fv, depth), axis=-1).astype(np.float32)
    pts = np.einsum('ik, vuk -> vui', pose[:3, :3], X) + pose[:3, 3][None, None, :]
    return pts, (depth > 0.0) & np.isfinite(pts).all(axis=-1)


def views_oracle(frames, resolution, rng, idx=0, ar_idx=0, aug_crop=False):
    views = []
    for v, f in enumerate(frames):
        pil, depth, K = crop_resize(f['img'], f['depthmap'], f['camera_intrinsics'], tuple(resolution), rng, aug_crop)
        pose = f['camera_pose'] if 'camera_pose' in f else np.full((4, 4), np.nan, dtype=np.float32)
        width, height = pil.size
        view = dict(img=_img_norm(pil), depthmap=depth, camera_intrinsics=K, camera_pose=pose, idx=(idx, ar_idx, v),
                    true_shape=np.int32((height, width)))
        view['pts3d'], view['valid_mask'] = unproject(depth, K, pose)
        views.append(view)
    for view in views:
        height, width = view['true_shape']
        if width < height:
            view['img'] = view['img'].swapaxes(1, 2)
            for k in ('depthmap', 'valid_mask'):
                view[k] = view[k].swapaxes(0, 1)
            view['pts3d'] = view['pts3d'].swapaxes(0, 1)
            view['camera_intrinsics'] = view['camera_intrinsics'][[1, 0, 2]]
        view['rng'] = int.from_bytes(rng.bytes(4), 'big')
    return views
