"""ctypes binding of libdust3r_b200.so (the C ABI declared in include/dust3r_b200.h).

There is deliberately NO fallback: if the shared library is missing or the device is not an H100
(sm_90), every compute entry point raises.  Build with `python -m dust3r_b200.build`.
"""
from __future__ import annotations

import ctypes as C
import os

from ._lib_fwd import Model

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


class JpegHuff(C.Structure):
    """Mirror of `d3r_jpeg_huff` (include/dust3r_b200.h)."""
    _fields_ = [('maxcode', C.c_int32 * 18), ('valoff', C.c_int32 * 18), ('look', C.c_uint16 * 512), ('val', C.c_uint8 * 256)]


class JpegDesc(C.Structure):
    """Mirror of `d3r_jpeg_desc` (include/dust3r_b200.h)."""
    _fields_ = [
        ('width', C.c_int32), ('height', C.c_int32), ('n_comp', C.c_int32), ('restart_interval', C.c_int32),
        ('orientation', C.c_int32), ('reserved', C.c_int32), ('scan_begin', C.c_int64),
        ('h_samp', C.c_int32 * 3), ('v_samp', C.c_int32 * 3), ('dc_table', C.c_int32 * 3), ('ac_table', C.c_int32 * 3),
        ('quant', (C.c_uint16 * 64) * 3), ('huff', JpegHuff * 8),
    ]


class PngDesc(C.Structure):
    """Mirror of `d3r_png_desc` (include/dust3r_b200.h)."""
    _fields_ = [
        ('width', C.c_int32), ('height', C.c_int32), ('color_type', C.c_int32), ('orientation', C.c_int32),
        ('palette_len', C.c_int32), ('reserved', C.c_int32), ('idat_bytes', C.c_int64), ('palette', (C.c_uint8 * 3) * 256),
    ]


class ViewDesc(C.Structure):
    """Mirror of `d3r_view_desc` (include/dust3r_b200.h)."""
    _fields_ = [
        ('src', C.c_void_p), ('depth', C.c_void_p), ('src_pitch', C.c_int32), ('depth_pitch', C.c_int32),
        ('H0', C.c_int32), ('W0', C.c_int32), ('H1', C.c_int32), ('W1', C.c_int32), ('crop_x0', C.c_int32), ('crop_y0', C.c_int32),
        ('H2', C.c_int32), ('W2', C.c_int32), ('row0', C.c_int32), ('rows', C.c_int32), ('transpose', C.c_int32),
        ('reserved', C.c_int32), ('xbounds', C.c_void_p), ('xcoefs', C.c_void_p), ('ybounds', C.c_void_p), ('ycoefs', C.c_void_p),
        ('fu', C.c_float), ('fv', C.c_float), ('cu', C.c_float), ('cv', C.c_float), ('pose', C.c_float * 12),
        ('tmp', C.c_void_p), ('img', C.c_void_p), ('depthmap', C.c_void_p), ('pts3d', C.c_void_p), ('valid', C.c_void_p),
        ('blocks', C.c_int64 * 3),
    ]


vp, i32, i64, u32, f32, f64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_float, C.c_double
_DESC, _MODEL, _JPEG, _PNG, _VIEW = (C.POINTER(AlignDesc), C.POINTER(Model), C.POINTER(JpegDesc), C.POINTER(PngDesc),
                                     C.POINTER(ViewDesc))

# restype, argtypes of every function include/dust3r_b200.h declares, in its order (tests/test_c_abi.py checks the two agree).
PROTOTYPES = {
    'd3r_last_error': (C.c_char_p, []),
    'd3r_abi_version': (i32, []),
    'd3r_check_device': (i32, []),
    'd3r_launch_count': (i64, []),
    'd3r_launch_count_reset': (None, []),
    'd3r_prof_enable': (None, [i32]),
    'd3r_prof_report': (i32, [C.c_char_p, i32]),
    'd3r_prof_dump': (i32, [C.c_char_p, i32]),
    # global alignment
    'd3r_sizeof_align_desc': (i32, []),
    'd3r_sizeof_align_item': (i32, []),
    'd3r_align_chunk_pixels': (i32, []),
    'd3r_align_workspace_floats': (i64, [i32, i32]),
    'd3r_align_prepare': (i32, [_DESC, vp]),
    'd3r_align_run': (i32, [_DESC, i32, i32, vp]),
    'd3r_align_pixel_pass': (i32, [_DESC, i32, vp]),
    'd3r_align_small_step': (i32, [_DESC, i32, vp]),
    'd3r_align_reduce_block': (i32, [i32, i32, C.POINTER(i64), C.POINTER(i64)]),
    'd3r_align_grad_pixel_pass': (i32, [_DESC, vp, vp]),
    'd3r_align_grad_small_step': (i32, [_DESC, vp, vp, vp]),
    'd3r_align_loss_grad': (i32, [_DESC, vp, vp, vp, vp]),
    'd3r_align_overflow_flag': (i32, [_DESC, C.POINTER(i32), vp]),
    'd3r_align_pts3d': (i32, [_DESC, vp, vp]),
    'd3r_align_set_debug': (i32, [vp]),
    'd3r_sizeof_pack_entry': (i32, []),
    'd3r_align_stream_slots_per_item': (i32, []),
    'd3r_align_stream_warps_per_cta': (i32, []),
    'd3r_align_stream_max_window': (i32, []),
    'd3r_align_pack_entries': (i32, [vp, i32, i32, i32, i32, vp, vp]),
    # forward building blocks
    'd3r_gemm_bf16': (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, i64, u32, vp, vp, i32, i32, i32, vp]),
    'd3r_conv3x3_bf16': (i32, [vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, u32, vp]),
    'd3r_attention_hd64': (i32, [vp, i64, vp, i64, vp, i64, vp, i64, i32, i32, i32, i32, f32, vp]),
    'd3r_conv_transpose_bf16': (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]),
    'd3r_conv3x3_head_tail': (i32, [vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, f32, vp]),
    'd3r_layernorm_bf16': (i32, [vp, vp, vp, vp, i32, i32, f32, vp]),
    'd3r_upsample2x_bf16': (i32, [vp, vp, i32, i32, i32, i32, i32, i32, vp]),
    'd3r_im2col_3x3_s2_bf16': (i32, [vp, vp, i32, i32, i32, i32, vp]),
    'd3r_patch_im2col16': (i32, [vp, vp, i32, i32, i32, vp]),
    'd3r_linear_head_postprocess': (i32, [vp, vp, vp, i32, i32, i32, i32, i32, i32, f32, f32, vp]),
    'd3r_set_gemm_impl': (None, [i32]),
    'd3r_set_gemm_store': (None, [i32]),
    'd3r_set_conv_store': (None, [i32]),
    'd3r_set_attention_impl': (None, [i32]),
    # scene-level operators
    'd3r_clean_pointcloud': (i32, [i32, vp, vp, i32, vp, vp, vp, vp, vp, f32, f32, vp]),
    'd3r_procrustes_moments': (i32, [i32, i32, vp, vp, vp, vp, vp]),
    'd3r_weiszfeld_focal': (i32, [i32, i32, i32, vp, vp, i32, vp, vp]),
    'd3r_nearest_neighbours': (i32, [i32, i32, vp, vp, vp, vp]),
    'd3r_image_resize_crop_normalize': (i32, [vp, i32, i32, i32, i32, vp, vp, i32, vp, vp, i32, i32, i32, i32, i32, i32, i32,
                                              vp, vp, vp, vp]),
    'd3r_sizeof_view_desc': (i32, []),
    'd3r_prepare_views': (i32, [i32, _VIEW, vp, vp, vp]),
    'd3r_sizeof_jpeg_desc': (i32, []),
    'd3r_jpeg_decode_workspace_bytes': (i64, [_JPEG, i64]),
    'd3r_jpeg_decode': (i32, [_JPEG, vp, i64, vp, vp, vp, i64, vp]),
    'd3r_sizeof_png_desc': (i32, []),
    'd3r_png_decode_workspace_bytes': (i64, [_PNG, i64]),
    'd3r_png_decode': (i32, [_PNG, vp, i64, vp, vp, vp, i64, vp]),
    'd3r_segment_sky_workspace_bytes': (i64, [i32, i64]),
    'd3r_segment_sky': (i32, [i32, vp, vp, i32, i64, vp, vp, vp, i64, vp]),
    'd3r_nanmedian_workspace_bytes': (i64, [i32]),
    'd3r_segmented_nanmedian': (i32, [i32, i64, vp, vp, vp, i64, vp]),
    'd3r_criterion_workspace_bytes': (i64, [i32, i64, i64, i32]),
    'd3r_criterion': (i32, [i32, i64, i64, i32, i32, f32, f32] + [vp] * 15 + [i64, vp]),
    'd3r_pnp_ransac_workspace_bytes': (i64, [i32]),
    'd3r_pnp_ransac': (i32, [i32, vp, vp, f64, f64, f64, f64, f64, f64, i32, i64, vp, i64, vp, vp, vp, vp]),
    'd3r_pnp_hypotheses': (i32, [i32, vp, vp, f64, f64, f64, f64, f64, i64, i32, i32, vp, vp, vp, vp]),
    # pairwise forward
    'd3r_sizeof_model': (i32, []),
    'd3r_encode_workspace_bytes': (i64, [_MODEL, i32, i32, i32]),
    'd3r_encode_images': (i32, [_MODEL, vp, i32, i32, i32, vp, vp, i64, vp]),
    'd3r_decode_workspace_bytes': (i64, [_MODEL, i32, i32, i32, i32, i32]),
    'd3r_decode_pairs': (i32, [_MODEL, vp, i32, i32, i32, vp, i32, i32, i32, C.POINTER(i32), C.POINTER(i32), i32,
                               vp, vp, vp, vp, vp, i64, vp]),
    'd3r_forward_set_debug': (i32, [i32, vp, i64]),
}


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
        for name, (restype, argtypes) in PROTOTYPES.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
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


def cuda_device(device):
    """require_cuda_device, with a bare 'cuda' resolved to the current device: the device tensors and caches are keyed on."""
    import torch
    dev = require_cuda_device(device)
    return torch.device('cuda', torch.cuda.current_device()) if dev.index is None else dev


def launch(device, name, *args):
    """Calls the entry point `name` with `args` and the current stream of `device`, with `device` current, and raises
    D3RError when it fails.  The stream is `device`'s, never the current device's: a scene on cuda:1 runs while cuda:0 is
    current."""
    import torch
    with torch.cuda.device(device):
        check(getattr(get_lib(), name)(*args, C.c_void_p(torch.cuda.current_stream(device).cuda_stream)))


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
