"""Restatement of segment_sky (dust3r/viz.py:345-381) for the parity tests of the sky kernels, built from library calls that do
not share code with the product's host path: OpenCV for the 8-bit HSV, scipy.ndimage for the opening and for an independent
8-connected labelling (the product's host path uses OpenCV's connectedComponentsWithStats).

  1. q = uint8(255 * clip(image, 0, 1)) (float32 product, truncation), uint8 input as is
  2. H, S, V = cv2.cvtColor(q, COLOR_BGR2HSV): the RGB array converted as BGR
  3. candidate = (H <= 30 & V >= 100) | (S < 10 & V > 150) | (S < 30 & V > 180) | (S < 50 & V > 220)
  4. binary opening with a 5x5 square, zero border
  5. 8-connected components; keep those with 2 * area > largest area
"""
import numpy as np


def quantise(image):
    image = np.asarray(image)
    return np.uint8(255 * image.clip(0, 1)) if np.issubdtype(image.dtype, np.floating) else image


def hsv(image):
    import cv2
    return cv2.cvtColor(np.ascontiguousarray(quantise(image)), cv2.COLOR_BGR2HSV)


def candidate(image):
    h, s, v = (hsv(image)[..., k].astype(np.int32) for k in range(3))
    return ((h <= 30) & (v >= 100)) | ((s < 10) & (v > 150)) | ((s < 30) & (v > 180)) | ((s < 50) & (v > 220))


def opened(image):
    from scipy import ndimage
    return ndimage.binary_opening(candidate(image), structure=np.ones((5, 5), dtype=bool), border_value=0)


def segment_sky(image):
    """(H, W, 3) RGB numpy image -> (H, W) bool numpy mask."""
    from scipy import ndimage
    fg = opened(image)
    labels, n = ndimage.label(fg, structure=np.ones((3, 3), dtype=int))
    if n == 0:
        return np.zeros(fg.shape, dtype=bool)
    area = np.bincount(labels.ravel(), minlength=n + 1)
    area[0] = 0
    return (2 * area > area.max())[labels]
