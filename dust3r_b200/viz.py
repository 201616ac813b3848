"""`segment_sky` of dust3r/viz.py:345-381, the one function of the reference's visualisation module the scene uses
(BasePCOptimizer.mask_sky).  The rest of that module (trimesh scenes, GLB export) is not part of this package.

A CUDA tensor goes to the batched kernel (`d3r_segment_sky`, csrc/sky_ops.cu, through cloud_opt/scene_ops.py); a numpy array
or a CPU tensor takes the host path below, OpenCV + scipy as in the reference.  Both give the reference's bits."""
from __future__ import annotations

import numpy as np
import torch


def _sky_host(image):
    """(H, W, 3) RGB numpy array (float in [0, 1] or uint8) -> (H, W) bool numpy mask."""
    import cv2
    from scipy import ndimage
    q = np.uint8(255 * image.clip(min=0, max=1)) if np.issubdtype(image.dtype, np.floating) else image
    # the reference converts its RGB array as BGR: channel 0 plays blue in the hue
    h, s, v = np.moveaxis(cv2.cvtColor(np.ascontiguousarray(q), cv2.COLOR_BGR2HSV).astype(np.int32), -1, 0)
    cand = ((h <= 30) & (v >= 100)) | ((s < 10) & (v > 150)) | ((s < 30) & (v > 180)) | ((s < 50) & (v > 220))
    fg = ndimage.binary_opening(cand, structure=np.ones((5, 5), dtype=bool))
    _, labels, stats, _ = cv2.connectedComponentsWithStats(fg.view(np.uint8), connectivity=8)
    area = stats[:, cv2.CC_STAT_AREA].astype(np.int64)
    area[0] = 0                                   # label 0 is the background
    keep = 2 * area > area.max()                  # every component larger than half the largest one (none for an empty mask)
    return keep[labels]


def segment_sky(image):
    """Sky mask of one (H, W, 3) RGB image: float in [0, 1] (an entry of scene.imgs) or uint8, as a numpy array or a tensor.
    Returns an (H, W) bool tensor on the input's device (the reference returns a CPU tensor)."""
    if torch.is_tensor(image) and image.is_cuda:
        from .cloud_opt.scene_ops import segment_sky as segment_sky_cuda
        return segment_sky_cuda([image])[0]
    arr = image.detach().cpu().numpy() if torch.is_tensor(image) else np.asarray(image)
    return torch.from_numpy(_sky_host(arr))
