"""Image I/O on the edges of the two hot paths: `load_images` builds the view dicts `inference()` consumes and `rgb`
turns normalised tensors back into displayable arrays for the optimizer's `imgs` attribute.  The conventions (long edge ->
`size`, dimensions cropped to multiples of 16, 4:3 crop of square inputs, [-1, 1] range, `true_shape`, `idx`, `instance`)
are those of dust3r/utils/image.py:74-128.

`load_images(..., device=None)` is the reference's host path (PIL resize + crop on a CPU core, float image to be uploaded by
inference()).  `load_images(..., device='cuda')` (SURVEY §8f rank 4) only DECODES on the host: the 8-bit RGB pixels go up once
and the resize (Pillow's two-pass fixed-point resampling, restated as two integer kernels), the crop and ImgNorm run on the
H100 (`d3r_image_resize_crop_normalize`, csrc/image_ops.cu) -- bit-identical to the host path, the normalised image is born
in HBM and inference() uses it in place."""
from __future__ import annotations

import ctypes
import functools
import math
import os

import numpy as np
import torch

_EXTENSIONS = ('.jpg', '.jpeg', '.png')


def rgb(ftensor, true_shape=None):
    """Normalised image(s) -> float arrays in [0, 1], channels last.  Accepts a tensor / array (CHW, BCHW or already
    channels-last), uint8 or [-1, 1] float data, or a list of those; `true_shape` = (H, W) crops the result."""
    if isinstance(ftensor, list):
        return [rgb(item, true_shape=true_shape) for item in ftensor]
    arr = ftensor.detach().cpu().numpy() if torch.is_tensor(ftensor) else np.asarray(ftensor)
    if arr.ndim == 3 and arr.shape[0] == 3:
        arr = np.moveaxis(arr, 0, -1)
    elif arr.ndim == 4 and arr.shape[1] == 3:
        arr = np.moveaxis(arr, 1, -1)
    if true_shape is not None:
        height, width = true_shape
        arr = arr[:height, :width]
    arr = arr.astype(np.float32) / 255 if arr.dtype == np.uint8 else arr * 0.5 + 0.5
    return arr.clip(min=0, max=1)


def img_to_arr(img):
    """A path is opened as RGB uint8; arrays pass through."""
    if isinstance(img, str):
        import PIL.Image
        return np.asarray(PIL.Image.open(img).convert('RGB'))
    return img


def _rescale(img, long_edge):
    """Resize so that the long edge becomes `long_edge` (Lanczos when shrinking, bicubic when enlarging)."""
    import PIL.Image
    current = max(img.size)
    method = PIL.Image.LANCZOS if current > long_edge else PIL.Image.BICUBIC
    return img.resize(tuple(int(round(side * long_edge / current)) for side in img.size), method)


def _crop_box(width, height, size, square_ok, patch_size=16):
    """Centre crop: a square for the 224 models, otherwise both sides rounded down to multiples of the patch size (and a
    square image cut to 4:3 unless square_ok)."""
    cx, cy = width // 2, height // 2
    if size == 224:
        half_w = half_h = min(cx, cy)
    else:
        half_w, half_h = ((2 * cx) // patch_size) * patch_size / 2, ((2 * cy) // patch_size) * patch_size / 2
        if width == height and not square_ok:
            half_h = 3 * half_w / 4
    return (cx - half_w, cy - half_h, cx + half_w, cy + half_h)


def _crop_box_int(width, height, size, square_ok, patch_size=16):
    """The box PIL.Image.crop really cuts: every coordinate rounded with Python's round()."""
    return tuple(int(round(v)) for v in _crop_box(width, height, size, square_ok, patch_size))


def _open_rgb(path):
    import PIL.Image
    from PIL.ImageOps import exif_transpose
    return exif_transpose(PIL.Image.open(path)).convert('RGB')


def _host_view(pil, size, square_ok, patch_size):
    """The reference's per-image pipeline on a decoded PIL image: resize, centre crop, ImgNorm -> (1, 3, H, W) CPU tensor."""
    w_in, h_in = pil.size
    # 224 models: the SHORT edge becomes 224 (then a square crop); the others: the long edge becomes `size`
    long_edge = round(size * max(w_in / h_in, h_in / w_in)) if size == 224 else size
    pil = _rescale(pil, long_edge)
    pil = pil.crop(_crop_box(pil.size[0], pil.size[1], size, square_ok, patch_size))
    pixels = torch.from_numpy(np.asarray(pil, dtype=np.float32) / 255).permute(2, 0, 1)
    return ((pixels - 0.5) / 0.5)[None]


def load_images(folder_or_list, size, square_ok=False, verbose=True, patch_size=16, device=None, workers=None):
    """Folder name or list of file names -> list of dict(img (1,3,H,W) in [-1,1], true_shape int32 [[H,W]], idx,
    instance) ready for make_pairs / inference.  Files that are not .jpg/.jpeg/.png are skipped.
    device=None: the reference's host pipeline, `img` is a CPU tensor.  device=<an H100>: decode on the host, resize / crop /
    normalise on that GPU (same bits), `img` is resident there.
    Files are decoded (device=None: decoded, resized and normalised) by `workers` threads -- PIL releases the GIL in its codecs
    and resampling loops -- while the results are consumed in file order, so idx / instance / verbose output are those of the
    reference's sequential loop; default min(8, cores), workers=1 is strictly sequential."""
    if isinstance(folder_or_list, str):
        root, names = folder_or_list, sorted(os.listdir(folder_or_list))
    elif isinstance(folder_or_list, list):
        root, names = '', folder_or_list
    else:
        raise ValueError(f'bad {folder_or_list=} ({type(folder_or_list)})')
    names = [name for name in names if name.lower().endswith(_EXTENSIONS)]

    def host_stage(name):
        pil = _open_rgb(os.path.join(root, name))
        if device is None:
            return pil.size, _host_view(pil, size, square_ok, patch_size)
        return pil.size, np.array(pil, dtype=np.uint8)

    if workers is None:
        workers = min(8, os.cpu_count() or 1)
    workers = max(1, min(int(workers), len(names)))
    views = []

    def consume(name, staged):
        (w_in, h_in), item = staged
        img = item if device is None else preprocess_image_u8(item, size, square_ok, device, patch_size)
        h_out, w_out = int(img.shape[-2]), int(img.shape[-1])
        if verbose:
            print(f' - adding {name} with resolution {w_in}x{h_in} --> {w_out}x{h_out}')
        views.append(dict(img=img, true_shape=np.int32([[h_out, w_out]]), idx=len(views), instance=str(len(views))))

    if workers == 1:
        for name in names:
            consume(name, host_stage(name))
    else:
        # at most 2 x workers files in flight (a decoded 12 Mpx photograph is 36 MB), consumed strictly in file order
        from collections import deque
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=workers) as pool:
            window, todo = deque(), iter(names)
            for name in todo:
                window.append((name, pool.submit(host_stage, name)))
                if len(window) >= 2 * workers:
                    first, fut = window.popleft()
                    consume(first, fut.result())
            while window:
                first, fut = window.popleft()
                consume(first, fut.result())
    assert views, 'no images found at ' + root
    if verbose:
        print(f' (Found {len(views)} images)')
    return views


# ------------------------------------------------------------------------------------------------------------------
# GPU preprocessing: host side of d3r_image_resize_crop_normalize
# ------------------------------------------------------------------------------------------------------------------
_PRECISION_BITS = 22        # Pillow Resample.c: 8-bit images use coefficients with 32 - 8 - 2 fractional bits
_LANCZOS, _BICUBIC = 'lanczos', 'bicubic'


def resized_shape(width, height, size):
    """(new width, new height, filter) of dust3r/utils/image.py:62-71 as load_images calls it (:101-106): Lanczos when the
    image shrinks, bicubic when it grows (or stays)."""
    long_edge = round(size * max(width / height, height / width)) if size == 224 else size
    current = max(width, height)
    method = _LANCZOS if current > long_edge else _BICUBIC
    return int(round(width * long_edge / current)), int(round(height * long_edge / current)), method


def _filter_weights(x, method):
    """Pillow's lanczos_filter (support 3) / bicubic_filter (a = -0.5, support 2) on a float64 array, evaluated with the C
    library's sin (math.sin) and the C expressions' operation order so that the rounded tables equal Pillow's."""
    if method == _BICUBIC:
        x = np.abs(x)
        near = ((-0.5 + 2.0) * x - (-0.5 + 3.0)) * x * x + 1
        far = (((x - 5) * x + 8) * x - 4) * -0.5
        return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))

    def sinc(v):
        v = v * math.pi
        return np.array([1.0 if t == 0.0 else math.sin(t) / t for t in v.ravel().tolist()], dtype=np.float64).reshape(v.shape)
    inside = (x >= -3.0) & (x < 3.0)
    return np.where(inside, sinc(x) * sinc(x / 3), 0.0)


@functools.lru_cache(maxsize=256)
def resample_table(in_size, out_size, method):
    """Pillow Resample.c precompute_coeffs + normalize_coeffs_8bpc for resizing `in_size` samples to `out_size` (whole-image
    box): (bounds int32 [out_size][2] = first source index and tap count, coefs int32 [out_size][ksize], 22 fractional
    bits).  An unchanged dimension gets the identity table (Pillow skips that pass; the fixed-point identity reproduces
    its input exactly)."""
    if in_size == out_size:
        bounds = np.stack([np.arange(out_size), np.ones(out_size, dtype=np.int64)], axis=1).astype(np.int32)
        return bounds, np.full((out_size, 1), 1 << _PRECISION_BITS, dtype=np.int32)
    scale = filterscale = float(in_size) / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = (3.0 if method == _LANCZOS else 2.0) * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    lo = np.trunc(center - support + 0.5).astype(np.int64)          # C int cast: truncation towards zero
    lo = np.maximum(lo, 0)
    hi = np.minimum(np.trunc(center + support + 0.5).astype(np.int64), in_size)
    cnt = hi - lo
    tap = np.arange(ksize, dtype=np.int64)[None, :]
    arg = ((tap + lo[:, None]) - center[:, None] + 0.5) * (1.0 / filterscale)
    w = np.where(tap < cnt[:, None], _filter_weights(arg, method), 0.0)
    total = np.add.accumulate(w, axis=1)[:, -1]                      # sequential sum, like the C loop (trailing zeros are neutral)
    k = np.where(total[:, None] != 0.0, w / np.where(total == 0.0, 1.0, total)[:, None], w)
    fixed = np.trunc(np.where(k < 0, -0.5, 0.5) + k * float(1 << _PRECISION_BITS)).astype(np.int64)
    return np.stack([lo, cnt], axis=1).astype(np.int32), fixed.astype(np.int32)


_DEVICE_TABLES = {}


def _device_table(dev, in_size, out_size, method):
    key = (dev, in_size, out_size, method)
    hit = _DEVICE_TABLES.get(key)
    if hit is None:
        if len(_DEVICE_TABLES) > 512:
            _DEVICE_TABLES.clear()
        bounds, coefs = resample_table(in_size, out_size, method)
        # the kernels read the coefficients tap-major ([ksize][out_size]): neighbouring threads, neighbouring words
        hit = (torch.from_numpy(bounds).to(dev), torch.from_numpy(np.ascontiguousarray(coefs.T)).to(dev), int(coefs.shape[1]))
        _DEVICE_TABLES[key] = hit
    return hit


def preprocess_plan(h0, w0, size, square_ok=False, patch_size=16):
    """The scalar arguments of d3r_image_resize_crop_normalize for a decoded image of h0 x w0: resized size and filter (which
    select the two coefficient tables), the crop window (left, upper, h2, w2) and the source rows [row0, row0 + rows) the
    cropped output reads."""
    w1, h1, method = resized_shape(w0, h0, size)
    left, upper, right, lower = _crop_box_int(w1, h1, size, square_ok, patch_size)
    w2, h2 = right - left, lower - upper
    if not (0 <= left and 0 <= upper and right <= w1 and lower <= h1 and w2 > 0 and h2 > 0):
        raise ValueError(f'image of {w0}x{h0} is too small for size={size}: crop box {(left, upper, right, lower)} of {w1}x{h1}')
    ybounds = resample_table(h0, h1, method)[0][upper:lower]
    row0 = int(ybounds[:, 0].min())
    rows = int((ybounds[:, 0] + ybounds[:, 1]).max()) - row0
    return dict(h1=h1, w1=w1, method=method, left=left, upper=upper, h2=h2, w2=w2, row0=row0, rows=rows)


def norm_lut():
    """The fp32 value of each of the 256 byte values after torchvision's ToTensor (x / 255) and Normalize ((x - 0.5) / 0.5),
    computed by the same torch CPU ops."""
    return torch.arange(256, dtype=torch.uint8).to(torch.float32).div(255).sub_(0.5).div_(0.5)


@torch.no_grad()
def preprocess_image_u8(pixels, size, square_ok=False, device='cuda', patch_size=16):
    """Decoded RGB image, uint8 (H, W, 3) numpy array or tensor (host or already on `device`) -> float32 (1, 3, H2, W2) on
    `device`, what load_images stores under 'img' for that picture: resize (long edge -> size; size 224: short edge -> 224),
    centre crop to multiples of 16 (224: square), x / 255 normalised to [-1, 1]."""
    from .. import _lib
    dev = _lib.require_cuda_device(device)
    if dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    src = torch.as_tensor(pixels)
    if src.dtype != torch.uint8 or src.ndim != 3 or src.shape[2] != 3:
        raise ValueError(f'preprocess_image_u8 expects uint8 (H, W, 3) RGB, got {src.dtype} {tuple(src.shape)}')
    h0, w0 = int(src.shape[0]), int(src.shape[1])
    plan = preprocess_plan(h0, w0, size, square_ok, patch_size)
    xb, xk, kx = _device_table(dev, w0, plan['w1'], plan['method'])
    yb, yk, ky = _device_table(dev, h0, plan['h1'], plan['method'])
    if (dev, 'lut') not in _DEVICE_TABLES:
        _DEVICE_TABLES[(dev, 'lut')] = norm_lut().to(dev)
    lut = _DEVICE_TABLES[(dev, 'lut')]
    src = src.contiguous().to(dev)
    tmp = torch.empty((plan['rows'], plan['w2'], 3), dtype=torch.uint8, device=dev)
    out = torch.empty((1, 3, plan['h2'], plan['w2']), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(_lib.get_lib().d3r_image_resize_crop_normalize(
            src.data_ptr(), h0, w0, plan['h1'], plan['w1'], xb.data_ptr(), xk.data_ptr(), kx, yb.data_ptr(), yk.data_ptr(), ky,
            plan['row0'], plan['rows'], plan['left'], plan['upper'], plan['h2'], plan['w2'], lut.data_ptr(), tmp.data_ptr(),
            out.data_ptr(), st))
    return out
