"""ctypes binding of libdust3r_b200.so (the C ABI declared in include/dust3r_b200.h).

There is deliberately NO fallback: if the shared library is missing or the device is not an H100
(sm_90), every compute entry point raises.  Build with `python -m dust3r_b200.build`.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libdust3r_b200.so')

_lib = None


class D3RError(RuntimeError):
    pass


class AlignDesc(C.Structure):
    """Mirror of `d3r_align_desc` (include/dust3r_b200.h)."""
    _fields_ = [
        ('n_imgs', C.c_int32), ('n_edges', C.c_int32), ('n_entries', C.c_int32), ('n_chunks', C.c_int32),
        ('max_deg', C.c_int32), ('max_chunks', C.c_int32), ('chunk_px', C.c_int32), ('dist_l2', C.c_int32), ('norm_pw_scale', C.c_int32),
        ('tied_focal', C.c_int32), ('eval_only', C.c_int32),
        ('base_scale', C.c_float), ('pw_break', C.c_float), ('focal_break', C.c_float), ('adam_eps', C.c_float),
        ('beta1', C.c_float), ('beta2', C.c_float),
        ('img_hw', C.c_void_p), ('img_pix_off', C.c_void_p), ('img_ent_ptr', C.c_void_p),
        ('img_chunk_ptr', C.c_void_p), ('chunk_img', C.c_void_p),
        ('ent_edge', C.c_void_p), ('ent_obs_off', C.c_void_p), ('ent_coef', C.c_void_p), ('edge_ent', C.c_void_p),
        ('obs', C.c_void_p),
        ('logd', C.c_void_p), ('logd_m', C.c_void_p), ('logd_v', C.c_void_p),
        ('small', C.c_void_p), ('small_m', C.c_void_p), ('small_v', C.c_void_p), ('small_trainable', C.c_void_p),
        ('workspace', C.c_void_p), ('sched', C.c_void_p), ('loss_out', C.c_void_p), ('counters', C.c_void_p),
        ('stream_kernel', C.c_int32), ('stream_grid', C.c_int32), ('stream_ppt', C.c_int32), ('stream_window', C.c_int32),
        ('n_items', C.c_int32), ('reserved0', C.c_int32), ('items', C.c_void_p), ('warp_item_ptr', C.c_void_p),
        ('items_rev', C.c_void_p), ('warp_item_ptr_rev', C.c_void_p),
    ]


def _declare(lib):
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    lib.d3r_last_error.restype = C.c_char_p
    lib.d3r_last_error.argtypes = []
    lib.d3r_abi_version.restype = C.c_int
    lib.d3r_check_device.restype = C.c_int
    lib.d3r_align_chunk_pixels.restype = C.c_int
    lib.d3r_launch_count.restype = C.c_longlong
    lib.d3r_launch_count_reset.restype = None
    lib.d3r_prof_enable.restype = None
    lib.d3r_prof_enable.argtypes = [C.c_int]
    lib.d3r_prof_report.restype = C.c_int
    lib.d3r_prof_report.argtypes = [C.c_char_p, C.c_int]
    lib.d3r_prof_dump.restype = C.c_int
    lib.d3r_prof_dump.argtypes = [C.c_char_p, C.c_int]
    lib.d3r_sizeof_align_desc.restype = C.c_int
    lib.d3r_align_workspace_floats.restype = i64
    lib.d3r_align_workspace_floats.argtypes = [i32, i32, i32, i32]
    for name in ('d3r_align_prepare',):
        getattr(lib, name).restype = C.c_int
        getattr(lib, name).argtypes = [C.POINTER(AlignDesc), vp]
    lib.d3r_align_run.restype = C.c_int
    lib.d3r_align_run.argtypes = [C.POINTER(AlignDesc), i32, i32, vp]
    lib.d3r_align_overflow_flag.restype = C.c_int
    lib.d3r_align_overflow_flag.argtypes = [C.POINTER(AlignDesc), C.POINTER(C.c_int32), vp]
    lib.d3r_align_pts3d.restype = C.c_int
    lib.d3r_align_pts3d.argtypes = [C.POINTER(AlignDesc), vp, vp]
    lib.d3r_align_pack_obs.restype = C.c_int
    lib.d3r_align_pack_obs.argtypes = [vp, vp, vp, i64, i64, vp]
    lib.d3r_align_pack_entries.restype = C.c_int
    lib.d3r_align_pack_entries.argtypes = [vp, i32, i32, i32, i32, vp, vp]
    lib.d3r_clean_pointcloud.restype = C.c_int
    lib.d3r_clean_pointcloud.argtypes = [i32, vp, vp, i32, vp, vp, vp, vp, vp, f32, f32, vp]
    lib.d3r_procrustes_moments.restype = C.c_int
    lib.d3r_procrustes_moments.argtypes = [i32, i32, vp, vp, vp, vp, vp]
    lib.d3r_weiszfeld_focal.restype = C.c_int
    lib.d3r_weiszfeld_focal.argtypes = [i32, i32, i32, vp, vp, i32, vp, vp]
    lib.d3r_nearest_neighbours.restype = C.c_int
    lib.d3r_nearest_neighbours.argtypes = [i32, i32, vp, vp, vp, vp]
    lib.d3r_image_resize_crop_normalize.restype = C.c_int
    lib.d3r_image_resize_crop_normalize.argtypes = [vp, i32, i32, i32, i32, vp, vp, i32, vp, vp, i32, i32, i32, i32, i32, i32, i32,
                                                    vp, vp, vp, vp]
    for name in ('d3r_sizeof_align_item', 'd3r_sizeof_pack_entry', 'd3r_align_stream_slots_per_item',
                 'd3r_align_stream_warps_per_cta', 'd3r_align_stream_max_window'):
        getattr(lib, name).restype = C.c_int
        getattr(lib, name).argtypes = []


def lib_available() -> bool:
    return os.path.exists(LIB_PATH)


def get_lib():
    """Loads the library (once).  Raises D3RError when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise D3RError(f'{LIB_PATH} not found: the CUDA extension is required (no CPU/torch fallback). '
                           f'Build it with `python -m dust3r_b200.build`.')
        lib = C.CDLL(LIB_PATH)
        _declare(lib)
        from . import _lib_fwd  # forward-path prototypes live next to their host code
        _lib_fwd.declare(lib)
        _lib = lib
    return _lib


def check(rc: int):
    if rc != 0:
        msg = get_lib().d3r_last_error().decode(errors='replace')
        raise D3RError(f'dust3r_b200 error {rc}: {msg}')


def require_cuda_device(device):
    """The product path only exists on an H100 (sm_90); fail loudly anywhere else."""
    import torch
    dev = torch.device(device)
    if dev.type != 'cuda':
        raise D3RError(f'dust3r_b200 computes on CUDA sm_90a only (got device {dev}); there is no CPU fallback')
    if not torch.cuda.is_available():
        raise D3RError('CUDA is not available: dust3r_b200 has no CPU fallback')
    with torch.cuda.device(dev):
        check(get_lib().d3r_check_device())
    return dev


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def launch_count(reset=False):
    lib = get_lib()
    n = int(lib.d3r_launch_count())
    if reset:
        lib.d3r_launch_count_reset()
    return n


def prof_enable(on=True):
    get_lib().d3r_prof_enable(1 if on else 0)


def prof_report():
    import json
    buf = C.create_string_buffer(1 << 16)
    n = get_lib().d3r_prof_report(buf, len(buf))
    if n < 0:
        raise D3RError('profile report does not fit the buffer')
    return json.loads(buf.value.decode())


def prof_dump():
    """Every launch recorded since prof_enable(True): [{tag, detail, ms, flops, bytes}] in launch order."""
    import json
    buf = C.create_string_buffer(1 << 22)
    n = get_lib().d3r_prof_dump(buf, len(buf))
    if n < 0:
        raise D3RError('profile dump does not fit the buffer')
    return json.loads(buf.value.decode())
