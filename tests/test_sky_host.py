"""Sky segmentation (`segment_sky`, dust3r/viz.py:345-381, and `mask_sky`, dust3r/cloud_opt/base_opt.py:289-295), CPU side:

  * the per-pixel colour test of the CUDA kernels (dust3r_b200/csrc/sky_core.h) is compiled for the HOST (tests/native/sky_host.cpp,
    g++) and checked on all 2^24 RGB triples against OpenCV's HSV and the reference's thresholds;
  * torch's device quantisation equals numpy's;
  * oracle/sky_oracle.py equals the unmodified reference's segment_sky (its outputs stored in tests/golden/segment_sky.npz);
  * the product's host path (dust3r_b200.viz.segment_sky) equals the oracle, and mask_sky on CPU scenes equals the reference's.
The `-m gpu` twin is tests/test_sky_gpu.py.  The image cases below are shared with it and with tests/golden/make_sky_golden.py.
"""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
import native_harness
from dust3r_b200.utils.synth import synth_consistent_scene, synth_pair_predictions, synth_sky_image
from oracle import sky_oracle

SKY, GROUND = (0.9, 0.9, 0.9), (0.1, 0.3, 0.1)      # a candidate (bright gray) and a non-candidate (dark green) colour


def _paint(mask):
    img = np.empty(mask.shape + (3,), dtype=np.float32)
    img[:] = GROUND
    img[mask] = SKY
    return img


def _serpentine(H, W, width, gap):
    """Horizontal bands of `width` rows joined at alternating ends: one long path."""
    m = np.zeros((H, W), dtype=bool)
    y, k = 2, 0
    while y + width <= H - 2:
        m[y:y + width, 2:W - 2] = True
        nxt = y + width + gap
        if nxt + width <= H - 2:
            x0 = W - 2 - width if k % 2 == 0 else 2
            m[y:nxt + width, x0:x0 + width] = True
        y, k = nxt, k + 1
    return m


def _spiral(H, W, width, gap):
    """Square spiral of `width`-wide arms, `gap` apart, walking inwards."""
    m = np.zeros((H, W), dtype=bool)
    top, left, bottom, right = 2, 2, H - 2, W - 2
    side = 0
    while bottom - top > width and right - left > width:
        if side == 0:
            m[top:top + width, left:right] = True
            top += width + gap
        elif side == 1:
            m[top - width - gap:bottom, right - width:right] = True
            right -= width + gap
        elif side == 2:
            m[bottom - width:bottom, left:right + width + gap] = True
            bottom -= width + gap
        else:
            m[top:bottom + width + gap, left:left + width] = True
            left += width + gap
        side = (side + 1) % 4
    return m


def _diagonal(H, W, block=5):
    """Checkerboard of block x block squares: after the opening they touch only at corners (one 8-connected component, many
    4-connected ones)."""
    yy, xx = np.meshgrid(np.arange(H) // block, np.arange(W) // block, indexing='ij')
    m = (yy + xx) % 2 == 0
    m[(H // block) * block:] = False
    m[:, (W // block) * block:] = False
    return m


def _rects(H, W, rects):
    m = np.zeros((H, W), dtype=bool)
    for y0, x0, h, w in rects:
        m[y0:y0 + h, x0:x0 + w] = True
    return m


def sky_cases():
    """name -> float32 (H, W, 3) RGB image in [0, 1]."""
    rng = np.random.default_rng(0)
    cases = {
        'synth_384x512_0': synth_sky_image(384, 512, seed=0),
        'synth_384x512_1': synth_sky_image(384, 512, seed=1),
        'synth_512x384': synth_sky_image(512, 384, seed=2),
        'synth_224x224': synth_sky_image(224, 224, seed=3),
        'synth_37x53': synth_sky_image(37, 53, seed=4),
        'noise_96x128': rng.random((96, 128, 3), dtype=np.float32),
        'black_64x80': np.zeros((64, 80, 3), dtype=np.float32),
        'white_64x80': np.ones((64, 80, 3), dtype=np.float32),
        'serpentine1px_96x128': _paint(_serpentine(96, 128, 1, 1)),
        'serpentine_121x160': _paint(_serpentine(121, 160, 5, 2)),
        'spiral_128x128': _paint(_spiral(128, 128, 5, 3)),
        'diagonal_62x71': _paint(_diagonal(62, 71)),
        # four bars along the four borders (areas 576, 456, 240, 240: the first two are kept)
        'borders_64x96': _paint(_rects(64, 96, [(0, 0, 6, 96), (58, 10, 6, 76), (12, 0, 40, 6), (12, 90, 40, 6)])),
        # two equal largest squares (both kept) and a smaller one
        'tied_64x96': _paint(_rects(64, 96, [(5, 5, 20, 20), (30, 60, 20, 20), (40, 10, 8, 8)])),
        # 400, exactly half of it (200, not kept), and 208 (kept)
        'half_64x96': _paint(_rects(64, 96, [(5, 5, 20, 20), (35, 5, 10, 20), (5, 50, 8, 26)])),
    }
    cases['uint8_37x53'] = np.uint8(255 * cases['synth_37x53'])
    return cases


def _views_with_images(out, imgs):
    """Adds the (3, H, W) [-1, 1] images of every pair to the view dicts, as load_images + inference leave them."""
    for view in ('view1', 'view2'):
        idx = out[view]['idx']
        out[view]['img'] = torch.stack([torch.from_numpy(2 * imgs[i] - 1).permute(2, 0, 1) for i in idx])
    return out


def sky_scene(kind):
    """Scene inputs (output of inference() plus images) of the mask_sky comparisons: 'pc' = 3 views, every ordered pair, for the
    optimizers; 'pv' = one symmetric pair of a consistent scene for PairViewer."""
    if kind == 'pc':
        n, H, W = 3, 48, 64
        out = synth_pair_predictions(n, [(i, j) for i in range(n) for j in range(n) if i != j], H, W, seed=7)
    else:
        n, H, W = 2, 48, 64
        out, _, _ = synth_consistent_scene(2, [(0, 1), (1, 0)], H, W, seed=3, noise=0.002)
    return _views_with_images(out, [synth_sky_image(H, W, seed=30 + i) for i in range(n)])


def golden():
    return np.load(os.path.join(GOLDEN, 'segment_sky.npz'))


def golden_mask(gold, name):
    shape = tuple(gold[f'img|{name}|shape'])
    return np.unpackbits(gold[f'img|{name}|bits'], count=int(np.prod(shape))).reshape(shape).astype(bool)


# ------------------------------------------------------------------------------------------------ the GPU colour test, on the host
@pytest.fixture(scope='module')
def host_colour():
    lib = ctypes.CDLL(native_harness.build('sky_host'))
    lib.sky_classify_host.restype = ctypes.c_int
    lib.sky_classify_host.argtypes = [ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def test_colour_test_on_every_rgb_triple_equals_opencv(host_colour):
    """sky_core.h (what the candidate kernel runs) vs cv2.cvtColor(COLOR_BGR2HSV) + the reference's thresholds, all 2^24 colours."""
    import cv2
    i = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(i >> 16) & 255, (i >> 8) & 255, i & 255], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)
    hsv = np.empty_like(rgb)
    cand = np.empty((4096, 4096), dtype=np.uint8)
    assert host_colour.sky_classify_host(rgb.ctypes.data, 1 << 24, hsv.ctypes.data, cand.ctypes.data) == 0
    ref = cv2.cvtColor(rgb, cv2.COLOR_BGR2HSV)
    for k in range(3):
        assert np.array_equal(hsv[..., k], ref[..., k]), 'HSV'[k]
    h, s, v = (ref[..., k].astype(np.int32) for k in range(3))
    want = ((h <= 30) & (v >= 100)) | ((s < 10) & (v > 150)) | ((s < 30) & (v > 180)) | ((s < 50) & (v > 220))
    assert np.array_equal(cand.astype(bool), want)
    assert 0.1 < want.mean() < 0.3


def test_torch_quantisation_equals_numpy():
    """(255 * x.clamp(0, 1)).to(uint8), as the CUDA path quantises, against np.uint8(255 * x.clip(0, 1)) of the reference."""
    from dust3r_b200.cloud_opt.scene_ops import _quantise
    k = np.arange(256, dtype=np.float64)
    centres = np.concatenate([(k / 255).astype(np.float32), np.float32([0, 1])])
    near = [centres]                                    # every float32 within 4 ulps of them
    for direction in (np.float32(-np.inf), np.float32(np.inf)):
        x = centres
        for _ in range(4):
            x = np.nextafter(x, direction)
            near.append(x)
    x = np.concatenate(near + [np.float32([-0.0]), np.linspace(-0.1, 1.1, 1 << 20, dtype=np.float32)])
    assert np.isfinite(x).all()
    ours = _quantise(torch.from_numpy(x)).numpy()
    assert np.array_equal(ours, np.uint8(255 * x.clip(0, 1)))
    assert np.array_equal(ours, sky_oracle.quantise(x))
    assert len(np.unique(ours)) == 256


def test_oracle_equals_reference_outputs():
    gold = golden()
    cases = sky_cases()
    assert sorted(cases) == sorted(str(s) for s in gold['img|names'])
    for name, img in cases.items():
        ref = golden_mask(gold, name)
        assert np.array_equal(sky_oracle.segment_sky(img), ref), name
    # the cases do what their names say
    assert golden_mask(gold, 'black_64x80').sum() == 0 and golden_mask(gold, 'white_64x80').all()
    assert golden_mask(gold, 'serpentine1px_96x128').sum() == 0
    assert golden_mask(gold, 'tied_64x96').sum() == 800 and golden_mask(gold, 'half_64x96').sum() == 608
    for name in ('synth_384x512_0', 'synth_512x384', 'serpentine_121x160', 'spiral_128x128', 'diagonal_62x71'):
        assert golden_mask(gold, name).mean() > 0.2, name


def test_host_path_equals_oracle():
    from dust3r_b200.viz import segment_sky
    for name, img in sky_cases().items():
        want = sky_oracle.segment_sky(img)
        for arg in (img, torch.from_numpy(img)):
            got = segment_sky(arg)
            assert torch.is_tensor(got) and got.dtype == torch.bool and got.device.type == 'cpu'
            assert np.array_equal(got.numpy(), want), name


@pytest.mark.parametrize('mode', ['PointCloudOptimizer', 'ModularPointCloudOptimizer', 'PairViewer'])
def test_mask_sky_on_cpu_scene_equals_reference(mode):
    """im_conf of mask_sky() against the unmodified reference's mask_sky() on the same inputs (tests/golden/segment_sky.npz);
    the scene itself is unchanged."""
    from dust3r_b200.cloud_opt import global_aligner, GlobalAlignerMode
    gold = golden()
    kind = 'pv' if mode == 'PairViewer' else 'pc'
    torch.manual_seed(0)
    scene = global_aligner(copy.deepcopy(sky_scene(kind)), 'cpu', mode=getattr(GlobalAlignerMode, mode), verbose=False)
    before = [c.detach().clone() for c in scene.im_conf]
    masked = scene.mask_sky()
    assert type(masked) is type(scene) and masked is not scene
    n_sky = 0
    for i, (c, b) in enumerate(zip(masked.im_conf, before)):
        ref = torch.from_numpy(gold[f'scene|{kind}|im_conf|{i}'])
        assert torch.equal(c.detach(), ref), i
        n_sky += int((c == 0).sum())
    assert n_sky > 100
    for c, b in zip(scene.im_conf, before):
        assert torch.equal(c.detach(), b)
    scene.imgs = None
    with pytest.raises(ValueError):
        scene.mask_sky()
