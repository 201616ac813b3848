"""Small host-side helpers of the forward path.

Only `is_symmetrized` carries reference semantics that the forward depends on (dust3r/utils/misc.py:32-40
decides, from the `instance` strings of a batch, whether it has the layout [(a,b),(b,a),(c,d),(d,c),...] whose
encoder work can be halved).  The head wrappers of the reference (`transpose_to_landscape`) have no counterpart here:
token-grid handling lives inside the C calls (`d3r_encode_images`, `d3r_decode_pairs`)."""
from __future__ import annotations

import inspect

import torch


def is_symmetrized(view1, view2) -> bool:
    """A batch is symmetrised when consecutive pairs mirror each other: instance1[2k] == instance2[2k+1] and
    instance1[2k+1] == instance2[2k] for every k.  One pair alone never counts.  An odd batch whose complete couples
    all mirror runs off the end in the reference (IndexError); that quirk is kept, a mismatch found earlier simply
    answers False."""
    first, second = view1['instance'], view2['instance']
    n = len(first)
    if n == len(second) == 1:
        return False
    for k in range(0, n, 2):
        if k + 1 >= n:
            raise IndexError('is_symmetrized: odd batch of mirrored couples')
        if first[k] != second[k + 1] or first[k + 1] != second[k]:
            return False
    return True


def freeze_all_params(modules) -> None:
    """requires_grad = False on every parameter of the given modules (plain tensors/parameters are accepted too)."""
    for mod in modules:
        params = mod.parameters() if isinstance(mod, torch.nn.Module) else [mod]
        for prm in params:
            prm.requires_grad_(False)


def fill_default_args(kwargs: dict, func) -> dict:
    """Complete `kwargs` in place with the defaults declared by `func`'s signature."""
    defaults = {name: prm.default for name, prm in inspect.signature(func).parameters.items()
                if prm.default is not inspect.Parameter.empty}
    for name, value in defaults.items():
        kwargs.setdefault(name, value)
    return kwargs


def interleave(x, y):
    """(x0,y0,x1,y1,...) and (y0,x0,y1,x1,...) along dim 0 -- how a batch is symmetrised on the fly."""
    n = x.shape[0]
    a = torch.empty((2 * n,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    b = torch.empty_like(a)
    a[0::2], a[1::2] = x, y
    b[0::2], b[1::2] = y, x
    return a, b


def invalid_to_nans(arr, valid_mask, ndim=999):
    """dust3r/utils/misc.py:103-109: a copy of `arr` with NaN where `valid_mask` is false (`arr` itself when the mask is None),
    its trailing spatial dimensions flattened so that it has at most `ndim` dimensions.  A uint8 mask counts as nonzero = valid."""
    if valid_mask is not None:
        arr = arr.clone()
        arr[~valid_mask.bool()] = float('nan')
    if arr.ndim > ndim:
        arr = arr.flatten(-2 - (arr.ndim - ndim), -2)
    return arr


def invalid_to_zeros(arr, valid_mask, ndim=999):
    """dust3r/utils/misc.py:112-121: (copy of `arr` with 0 where `valid_mask` is false, number of valid entries per batch item);
    without a mask, `arr` itself and the number of entries per item.  Trailing spatial dimensions flattened as invalid_to_nans."""
    if valid_mask is not None:
        valid_mask = valid_mask.bool()
        arr = arr.clone()
        arr[~valid_mask] = 0
        nnz = valid_mask.view(len(valid_mask), -1).sum(1)
    else:
        nnz = arr.numel() // len(arr) if len(arr) else 0
    if arr.ndim > ndim:
        arr = arr.flatten(-2 - (arr.ndim - ndim), -2)
    return arr, nnz
