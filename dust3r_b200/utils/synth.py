"""Deterministic synthetic weights / images / pointmaps.

There are no checkpoints or datasets offline, so tests, goldens and bench.py all draw from here.  Values
depend only on (key, shape, seed) through torch's CPU Philox-free default generator, which is
reproducible across machines for a fixed torch version; goldens additionally store the outputs.
"""
from __future__ import annotations

import hashlib
import math
import torch

from ..config import ModelConfig, state_dict_spec


def _gen(seed: int, key: str) -> torch.Generator:
    h = int.from_bytes(hashlib.sha256(f'{seed}:{key}'.encode()).digest()[:7], 'little')
    g = torch.Generator(device='cpu')
    g.manual_seed(h)
    return g


def synth_state_dict(cfg: ModelConfig, seed: int = 0, dtype=torch.float32):
    """Xavier-like weights (as croco.py:111-127 initialises them) but with non-zero biases and
    non-unit LayerNorm gains so every epilogue path is exercised.  layer_rn.k aliases layer{k+1}_rn."""
    sd = {}
    spec = state_dict_spec(cfg)
    for key, shape in spec.items():
        if '.scratch.layer_rn.' in key:
            continue
        g = _gen(seed, key)
        if key == 'mask_token':
            t = torch.randn(shape, generator=g) * 0.02
        elif '.norm' in key or key.startswith(('enc_norm', 'dec_norm')):
            if key.endswith('weight'):
                t = 1.0 + 0.1 * torch.randn(shape, generator=g)
            else:
                t = 0.05 * torch.randn(shape, generator=g)
        elif key.endswith('bias'):
            t = 0.02 * torch.randn(shape, generator=g)
        else:
            fan_out = shape[0] * (math.prod(shape[2:]) if len(shape) > 2 else 1)
            fan_in = math.prod(shape[1:])
            if '.act_postprocess.0.1.' in key or '.act_postprocess.1.1.' in key:
                # ConvTranspose2d weight is (Cin, Cout, k, k): every output pixel sees Cin taps
                fan_in, fan_out = shape[0], shape[1]
            a = math.sqrt(6.0 / (fan_in + fan_out))
            if key.endswith('.dpt.head.4.weight'):
                # un-normalised DPT trunk reaches std~8 with xavier weights; trained heads emit O(1)
                # log-depths, so damp the last 1x1 conv to keep exp()/expm1() in a sane range
                a *= 0.06
            t = (torch.rand(shape, generator=g) * 2 - 1) * a
        sd[key] = t.to(dtype)
    for key in spec:
        if '.scratch.layer_rn.' in key:
            k = int(key.split('.scratch.layer_rn.')[1].split('.')[0])
            sd[key] = sd[key.replace(f'.scratch.layer_rn.{k}.', f'.scratch.layer{k + 1}_rn.')]
    return {k: sd[k] for k in spec}


def synth_images(n: int, H: int, W: int, seed: int = 0):
    """n images in [-1,1] (the ImgNorm range, dust3r/utils/image.py:23) in load_images' dict format
    (utils/image.py:122-123)."""
    import numpy as np
    out = []
    for i in range(n):
        g = _gen(seed, f'img{i}')
        # smooth-ish content: low-res noise upsampled + fine noise, clipped to [-1,1]
        low = torch.rand((1, 3, max(H // 16, 1), max(W // 16, 1)), generator=g) * 2 - 1
        img = torch.nn.functional.interpolate(low, size=(H, W), mode='bilinear', align_corners=False)
        img = (img + 0.25 * (torch.rand((1, 3, H, W), generator=g) * 2 - 1)).clamp(-1, 1)
        out.append(dict(img=img, true_shape=np.int32([[H, W]]), idx=i, instance=str(i)))
    return out


def synth_pair_predictions(n_imgs: int, edges, H: int, W: int, seed: int = 0):
    """Directly synthesise what inference() would return for `edges` (list of (i,j)), as SURVEY §8d
    prescribes for the alignment benchmark: pts3d ~ N(0,1)+[0,0,3], conf = 1 + 5*U(0,1)."""
    E = len(edges)
    g = _gen(seed, f'pairs{n_imgs}:{E}:{H}x{W}')
    off = torch.tensor([0.0, 0.0, 3.0])
    pts1 = torch.randn((E, H, W, 3), generator=g) + off
    pts2 = torch.randn((E, H, W, 3), generator=g) + off
    conf1 = 1 + 5 * torch.rand((E, H, W), generator=g)
    conf2 = 1 + 5 * torch.rand((E, H, W), generator=g)
    import numpy as np
    ts = torch.from_numpy(np.int32([[H, W]] * E))
    view1 = dict(idx=[int(i) for i, j in edges], instance=[str(i) for i, j in edges], true_shape=ts)
    view2 = dict(idx=[int(j) for i, j in edges], instance=[str(j) for i, j in edges], true_shape=ts)
    pred1 = dict(pts3d=pts1, conf=conf1)
    pred2 = dict(pts3d_in_other_view=pts2, conf=conf2)
    return dict(view1=view1, view2=view2, pred1=pred1, pred2=pred2, loss=None)


def synth_consistent_scene(n_imgs: int, edges, H: int, W: int, seed: int = 0, noise: float = 0.01):
    """A geometrically consistent toy scene: smooth random depth maps seen by cameras on a small arc, exact
    pairwise pointmaps (image i's points in camera i's frame / image j's points in camera i's frame) plus
    a little noise, confidences in [1.5, 6].  Gives the initialisers (MST / PnP / Procrustes) something
    meaningful to recover, unlike synth_pair_predictions' white noise."""
    import numpy as np
    g = _gen(seed, f'scene{n_imgs}:{H}x{W}')
    f = 1.2 * max(H, W)
    vs, us = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing='ij')
    cams, clouds = [], []
    for i in range(n_imgs):
        low = torch.rand((1, 1, 4, 4), generator=g)
        depth = 2.0 + torch.nn.functional.interpolate(low, size=(H, W), mode='bicubic', align_corners=True)[0, 0]
        pts_cam = torch.stack(((us - W / 2) * depth / f, (vs - H / 2) * depth / f, depth), dim=-1)
        ang = 0.25 * (i - (n_imgs - 1) / 2)
        R = torch.tensor([[math.cos(ang), 0, math.sin(ang)], [0, 1, 0], [-math.sin(ang), 0, math.cos(ang)]], dtype=torch.float32)
        t = torch.tensor([1.5 * math.sin(ang), 0.05 * i, 0.3 * (1 - math.cos(ang))], dtype=torch.float32)
        c2w = torch.eye(4)
        c2w[:3, :3], c2w[:3, 3] = R, t
        cams.append(c2w)
        clouds.append(pts_cam)

    def to_frame(pts_cam, c2w_src, c2w_dst):
        world = pts_cam @ c2w_src[:3, :3].T + c2w_src[:3, 3]
        w2c = torch.linalg.inv(c2w_dst)
        return world @ w2c[:3, :3].T + w2c[:3, 3]
    p1, p2, c1, c2 = [], [], [], []
    for (i, j) in edges:
        p1.append(clouds[i] + noise * torch.randn((H, W, 3), generator=g))
        p2.append(to_frame(clouds[j], cams[j], cams[i]) + noise * torch.randn((H, W, 3), generator=g))
        c1.append(1.5 + 4.5 * torch.rand((H, W), generator=g))
        c2.append(1.5 + 4.5 * torch.rand((H, W), generator=g))
    ts = torch.from_numpy(np.int32([[H, W]] * len(edges)))
    out = dict(view1=dict(idx=[int(i) for i, j in edges], instance=[str(i) for i, j in edges], true_shape=ts),
               view2=dict(idx=[int(j) for i, j in edges], instance=[str(j) for i, j in edges], true_shape=ts),
               pred1=dict(pts3d=torch.stack(p1), conf=torch.stack(c1)),
               pred2=dict(pts3d_in_other_view=torch.stack(p2), conf=torch.stack(c2)), loss=None)
    return out, torch.stack(cams), f


def many_ar_inputs(H: int, W: int, seed: int = 9):
    """4 pairs stored in landscape (H x W, W >= H) for the landscape_only=True (ManyAR) path; orientation of
    (view1, view2) per item: LL, LP, PL, PP -- a portrait item is the transposed storage of a (W x H) image."""
    g = torch.Generator().manual_seed(seed)
    img1 = torch.rand((4, 3, H, W), generator=g) * 2 - 1
    img2 = torch.rand((4, 3, H, W), generator=g) * 2 - 1
    L, P = [H, W], [W, H]
    ts1 = torch.tensor([L, L, P, P], dtype=torch.int32)
    ts2 = torch.tensor([L, P, L, P], dtype=torch.int32)
    return (dict(img=img1, true_shape=ts1, instance=['0', '1', '2', '3']),
            dict(img=img2, true_shape=ts2, instance=['4', '5', '6', '7']))


def synth_sky_image(H: int, W: int, seed: int = 0):
    """An outdoor scene as scene.imgs holds it: float32 (H, W, 3) RGB in [0, 1].  A blue-to-hazy sky with bright clouds above a
    wavy horizon, textured dark ground below it with a few bright patches, sensor noise everywhere -- input of the sky
    segmentation tests and benchmark (sky, clouds and bright ground patches give components of many sizes)."""
    g = _gen(seed, f'sky{H}x{W}')
    y = torch.linspace(0, 1, H)[:, None]
    x = torch.linspace(0, 1, W)[None, :]
    ph = torch.rand((3,), generator=g) * 6.28
    horizon = 0.45 + 0.1 * torch.sin(6.28 * x + ph[0]) + 0.05 * torch.sin(17 * x + ph[1])
    t = (y / horizon).clamp(0, 1)[..., None]
    sky = (1 - t) * torch.tensor([0.25, 0.45, 0.85]) + t * torch.tensor([0.75, 0.8, 0.9])
    for _ in range(5):      # clouds: soft bright ellipses
        c = torch.rand((4,), generator=g)
        d = ((x - c[0]) / (0.05 + 0.15 * c[2])) ** 2 + ((y - 0.3 * c[1]) / (0.02 + 0.05 * c[3])) ** 2
        sky = sky + 0.5 * torch.exp(-d)[..., None]
    low = torch.rand((1, 3, max(H // 8, 1), max(W // 8, 1)), generator=g)
    tex = torch.nn.functional.interpolate(low, size=(H, W), mode='bilinear', align_corners=False)[0].permute(1, 2, 0)
    ground = torch.tensor([0.3, 0.25, 0.15]) + 0.25 * (tex - 0.5)
    for _ in range(3):      # bright patches on the ground (walls, snow): sky-coloured but not sky
        r = torch.rand((4,), generator=g)
        y0, x0 = int((0.6 + 0.3 * r[0]) * H), int(r[1] * W * 0.8)
        ground[y0:y0 + 2 + int(r[2] * H * 0.15), x0:x0 + 2 + int(r[3] * W * 0.2)] = 0.92
    img = torch.where((y < horizon)[..., None], sky, ground)
    img = img + 0.04 * torch.randn((H, W, 3), generator=g)
    return img.clamp(0, 1).numpy()


def synth_photo(H: int, W: int, seed: int = 0):
    """A decoded 'photograph': uint8 (H, W, 3) numpy array with natural-image statistics (smooth colour fields, a few hard
    edges, sensor noise) -- input of the load_images preprocessing tests (edges and noise exercise the negative lobes and the
    clipping of the resampling filters, which flat or purely random images do not)."""
    g = _gen(seed, f'photo{H}x{W}')
    y = torch.linspace(0, 1, H)[:, None, None]
    x = torch.linspace(0, 1, W)[None, :, None]
    f = torch.rand((6, 3), generator=g) * 9 + 1
    p = torch.rand((6, 3), generator=g) * 6.28
    field = sum(torch.sin(f[k] * (x if k % 2 else y) * 6.28 + p[k]) for k in range(6)) / 6
    img = 127 + 110 * field
    # hard-edged rectangles (saturated values next to dark ones: ringing gets clipped)
    for _ in range(4):
        r = torch.rand((4,), generator=g)
        y0, x0 = int(r[0] * H * 0.8), int(r[1] * W * 0.8)
        y1, x1 = y0 + 1 + int(r[2] * H * 0.3), x0 + 1 + int(r[3] * W * 0.3)
        img[y0:y1, x0:x1] = torch.randint(0, 2, (3,), generator=g).to(torch.float32) * 255
    img = img + torch.randn((H, W, 3), generator=g) * 12
    return img.clamp(0, 255).to(torch.uint8).numpy()


def synth_criterion_batch(B: int, hw1, hw2, seed: int = 0, invalid: float = 0.2, garbage: bool = True, empty_view2: bool = False,
                          noise: float = 0.02):
    """Ground truth and predictions for the evaluation criteria (dust3r_b200.losses): B pairs of views of sizes hw1 and hw2.
    Per pair, two cameras on a small arc look at smooth random depth maps; the views carry the world points 'pts3d', a
    'valid_mask' (a random `invalid` share of the pixels and a rectangular hole are invalid; all of view 2 with empty_view2)
    and the 'camera_pose' (camera to world).  The predictions are the exact points in camera 1's frame at a random scale per
    pair plus noise, with confidences in [1, 5].  With garbage, invalid ground truth holds NaN, +-Inf and 1e30, which must not
    reach any result.  Returns (gt1, gt2, pred1, pred2), CPU fp32."""
    g = _gen(seed, f'criterion{B}:{tuple(hw1)}:{tuple(hw2)}')

    def cam_points(H, W):
        f = 1.2 * max(H, W)
        vs, us = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing='ij')
        depth = 2.0 + torch.nn.functional.interpolate(torch.rand((1, 1, 4, 4), generator=g), size=(H, W), mode='bicubic',
                                                      align_corners=True)[0, 0]
        return torch.stack(((us - W / 2) * depth / f, (vs - H / 2) * depth / f, depth), dim=-1)

    def pose(ang, t):
        c2w = torch.eye(4)
        c2w[:3, :3] = torch.tensor([[math.cos(ang), 0, math.sin(ang)], [0, 1, 0], [-math.sin(ang), 0, math.cos(ang)]])
        c2w[:3, 3] = torch.tensor(t)
        return c2w

    def mask(H, W):
        m = torch.rand((H, W), generator=g) >= invalid
        y0, x0 = int(torch.randint(0, H // 2, (1,), generator=g)), int(torch.randint(0, W // 2, (1,), generator=g))
        m[y0:y0 + H // 4, x0:x0 + W // 4] = False
        return m

    views = ([], [], [], [], [], [], [], [])   # gt1, gt2, valid1, valid2, pose1, pose2, pred1, pred2
    for b in range(B):
        ang = 0.3 * float(torch.rand((), generator=g)) - 0.15
        c1 = pose(ang, [0.1 * b, 0.0, 0.0])
        c2 = pose(ang + 0.25, [0.1 * b + 0.6, 0.05, 0.1])
        p1, p2 = cam_points(*hw1), cam_points(*hw2)
        w1 = p1 @ c1[:3, :3].T + c1[:3, 3]
        w2 = p2 @ c2[:3, :3].T + c2[:3, 3]
        w2c1 = torch.linalg.inv(c1)
        p2_in_1 = w2 @ w2c1[:3, :3].T + w2c1[:3, 3]
        s = 0.5 + 1.5 * float(torch.rand((), generator=g))
        for k, v in enumerate((w1, w2, mask(*hw1), mask(*hw2), c1, c2,
                               s * p1 + noise * torch.randn(p1.shape, generator=g),
                               s * p2_in_1 + noise * torch.randn(p2.shape, generator=g))):
            views[k].append(v)
    gt1, gt2, v1, v2, pose1, pose2, pr1, pr2 = (torch.stack(v) for v in views)
    if empty_view2:
        v2[:] = False
    if garbage:
        junk = torch.tensor([float('nan'), float('inf'), -float('inf'), 1e30])
        for gt, v in ((gt1, v1), (gt2, v2)):
            bad = (~v).nonzero()
            gt[bad[:, 0], bad[:, 1], bad[:, 2]] = junk[torch.arange(len(bad)) % 4, None]
    conf1 = 1 + 4 * torch.rand(v1.shape, generator=g)
    conf2 = 1 + 4 * torch.rand(v2.shape, generator=g)
    return (dict(pts3d=gt1, valid_mask=v1, camera_pose=pose1), dict(pts3d=gt2, valid_mask=v2, camera_pose=pose2),
            dict(pts3d=pr1, conf=conf1), dict(pts3d_in_other_view=pr2, conf=conf2))


def synth_rgbd_frame(H: int, W: int, seed: int = 0, pp=None, pose: bool = True):
    """An RGB-D frame as a dataset hands it to the view stage (dust3r_b200.views): dict(img uint8 (H, W, 3) RGB, depthmap fp32
    (H, W), camera_intrinsics fp32 3x3 without skew, camera_pose fp32 4x4 camera-to-world, left out with pose=False).  `pp` =
    the principal point (default within 5 % of the centre).  The depth is a smooth positive field with a patch of zeros and one
    of negative values (both invalid).  Built from uniform draws with + - * / and sqrt only, so the bytes are the same on every
    machine and numpy build."""
    import numpy as np
    rng = np.random.default_rng([seed, H, W])
    y, x = np.arange(H, dtype=np.float64)[:, None], np.arange(W, dtype=np.float64)[None, :]
    u, v = x / max(W - 1, 1), y / max(H - 1, 1)
    col = rng.random((4, 3)) * 255
    img = (col[0] * (1 - u[..., None]) * (1 - v[..., None]) + col[1] * u[..., None] * (1 - v[..., None])
           + col[2] * (1 - u[..., None]) * v[..., None] + col[3] * u[..., None] * v[..., None])
    for _ in range(4):       # hard edges: saturated rectangles
        r = rng.random(4)
        y0, x0 = int(r[0] * H * 0.8), int(r[1] * W * 0.8)
        img[y0:y0 + 1 + int(r[2] * H * 0.3), x0:x0 + 1 + int(r[3] * W * 0.3)] = (rng.random(3) < 0.5) * 255.0
    img = img + (rng.random((H, W, 3)) - 0.5) * 24
    img = np.clip(np.floor(img), 0, 255).astype(np.uint8)
    a = rng.random(4)
    depth = 1.0 + 4 * a[0] + 2 * a[1] * u + 3 * a[2] * v * v + a[3] * u * v + 0.01 * rng.random((H, W))
    r = rng.random(4)
    depth[int(r[0] * H * 0.7):int(r[0] * H * 0.7) + 1 + H // 8, int(r[1] * W * 0.7):int(r[1] * W * 0.7) + 1 + W // 8] = 0.0
    depth[int(r[2] * H * 0.7):int(r[2] * H * 0.7) + 1 + H // 10, int(r[3] * W * 0.7):int(r[3] * W * 0.7) + 1 + W // 10] *= -1.0
    k = rng.random(4)
    f = (0.7 + 0.8 * k[0]) * max(H, W)
    cx, cy = pp if pp is not None else (W / 2 + (k[1] - 0.5) * 0.1 * W, H / 2 + (k[2] - 0.5) * 0.1 * H)
    K = np.array([[f, 0, cx], [0, f * (0.98 + 0.04 * k[3]), cy], [0, 0, 1]], dtype=np.float32)
    frame = dict(img=img, depthmap=depth.astype(np.float32), camera_intrinsics=K)
    if pose:
        q = rng.random(4) * 2 - 1
        q = q / np.sqrt((q * q).sum())
        a, b, c, d = q
        R = [[1 - 2 * (c * c + d * d), 2 * (b * c - a * d), 2 * (b * d + a * c)],
             [2 * (b * c + a * d), 1 - 2 * (b * b + d * d), 2 * (c * d - a * b)],
             [2 * (b * d - a * c), 2 * (c * d + a * b), 1 - 2 * (b * b + c * c)]]
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, rng.random(3) * 4 - 2
        frame['camera_pose'] = T.astype(np.float32)
    return frame
