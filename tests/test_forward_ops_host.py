"""The forward's building-block entry points reject bad arguments with D3R_ERR_INVALID and a message naming the op, before any
CUDA call or launch (no GPU needed: every call below fails its argument checks, so no pointer is ever dereferenced)."""
import ctypes

import pytest

D3R_ERR_INVALID = -1
P = 4096          # a 16-byte aligned stand-in for a device pointer
ODD = 4098        # a misaligned one
F_CONVT, F_HEAD_FINAL = 1 << 9, 1 << 10


@pytest.fixture(scope='module')
def lib():
    from dust3r_b200 import build, _lib
    build.build()
    return _lib.get_lib()


def _rejects(lib, rc, op):
    assert rc == D3R_ERR_INVALID, (op, rc)
    msg = lib.d3r_last_error().decode()
    assert msg.startswith(op + ':'), msg
    return msg


CASES = {
    'layernorm': [
        lambda L: L.d3r_layernorm_bf16(0, P, P, P, 8, 64, 1e-6, None),
        lambda L: L.d3r_layernorm_bf16(P, P, P, P, 0, 64, 1e-6, None),
        lambda L: L.d3r_layernorm_bf16(P, P, P, P, 8, 6, 1e-6, None),
        lambda L: L.d3r_layernorm_bf16(P, P, P, P, 8, 4096, 1e-6, None),
        lambda L: L.d3r_layernorm_bf16(ODD, P, P, P, 8, 64, 1e-6, None),
    ],
    'upsample2x': [
        lambda L: L.d3r_upsample2x_bf16(P, 0, 1, 4, 4, 128, 8, 8, None),
        lambda L: L.d3r_upsample2x_bf16(P, P, 0, 4, 4, 128, 8, 8, None),
        lambda L: L.d3r_upsample2x_bf16(P, P, 1, 4, 4, 128, 9, 8, None),
        lambda L: L.d3r_upsample2x_bf16(P, P, 1, 4, 4, 128, 8, 0, None),
        lambda L: L.d3r_upsample2x_bf16(P, P, 1, 4, 4, 24, 8, 8, None),
        lambda L: L.d3r_upsample2x_bf16(P, P, 1, 4, 4, 12, 8, 8, None),
        lambda L: L.d3r_upsample2x_bf16(P, ODD, 1, 4, 4, 128, 8, 8, None),
    ],
    'im2col_s2': [
        lambda L: L.d3r_im2col_3x3_s2_bf16(0, P, 1, 4, 4, 64, None),
        lambda L: L.d3r_im2col_3x3_s2_bf16(P, P, 1, 0, 4, 64, None),
        lambda L: L.d3r_im2col_3x3_s2_bf16(P, P, 1, 4, 4, 12, None),
        lambda L: L.d3r_im2col_3x3_s2_bf16(ODD, P, 1, 4, 4, 64, None),
    ],
    'patch_im2col': [
        lambda L: L.d3r_patch_im2col16(0, P, 1, 32, 32, None),
        lambda L: L.d3r_patch_im2col16(P, P, 0, 32, 32, None),
        lambda L: L.d3r_patch_im2col16(P, P, 1, 24, 32, None),
        lambda L: L.d3r_patch_im2col16(P, ODD, 1, 32, 32, None),
    ],
    'linear_head_postprocess': [
        lambda L: L.d3r_linear_head_postprocess(0, P, P, 1, 2, 2, 4, 0, 1, 1.0, 2.0, None),
        lambda L: L.d3r_linear_head_postprocess(P, P, P, 1, 0, 2, 4, 0, 1, 1.0, 2.0, None),
        lambda L: L.d3r_linear_head_postprocess(P, P, P, 1, 2, 2, 5, 0, 1, 1.0, 2.0, None),
        lambda L: L.d3r_linear_head_postprocess(P, P, P, 1, 2, 2, 4, 3, 1, 1.0, 2.0, None),
        lambda L: L.d3r_linear_head_postprocess(P, P, P, 1, 2, 2, 4, 0, -1, 1.0, 2.0, None),
        lambda L: L.d3r_linear_head_postprocess(P, P, 0, 1, 2, 2, 4, 0, 2, 1.0, 2.0, None),
    ],
    'conv_transpose': [
        lambda L: L.d3r_conv_transpose_bf16(0, P, P, P, 1, 4, 4, 96, 96, 4, None),
        lambda L: L.d3r_conv_transpose_bf16(P, P, P, P, 0, 4, 4, 96, 96, 4, None),
        lambda L: L.d3r_conv_transpose_bf16(P, P, P, P, 1, 4, 4, 96, 96, 0, None),
        lambda L: L.d3r_conv_transpose_bf16(P, P, P, P, 1, 4, 4, 12, 96, 4, None),
        lambda L: L.d3r_conv_transpose_bf16(P, P, P, P, 1, 4, 4, 96, 3, 8, None),     # k*k*Cout = 192, but Cout odd
        lambda L: L.d3r_conv_transpose_bf16(P, P, P, P, 1, 4, 4, 96, 10, 1, None),
    ],
    'conv3x3_head_tail': [
        lambda L: L.d3r_conv3x3_head_tail(P, P, P, 0, P, P, P, 1, 16, 16, 0, 1, 1.0, 2.0, None),
        lambda L: L.d3r_conv3x3_head_tail(P, P, P, P, P, P, P, 1, 0, 16, 0, 1, 1.0, 2.0, None),
        lambda L: L.d3r_conv3x3_head_tail(P, P, P, P, P, P, P, 1, 16, 16, 3, 1, 1.0, 2.0, None),
        lambda L: L.d3r_conv3x3_head_tail(P, P, P, P, P, P, P, 1, 16, 16, 0, 3, 1.0, 2.0, None),
        lambda L: L.d3r_conv3x3_head_tail(P, P, P, P, P, P, 0, 1, 16, 16, 0, 1, 1.0, 2.0, None),
    ],
}


@pytest.mark.parametrize('op', sorted(CASES))
def test_bad_arguments_are_rejected_before_device_work(lib, op):
    launches = lib.d3r_launch_count()
    for case in CASES[op]:
        _rejects(lib, case(lib), op)
    assert lib.d3r_launch_count() == launches


def test_gemm_points_to_the_dedicated_entry_points(lib):
    for flag in (F_CONVT, F_HEAD_FINAL):
        msg = _rejects(lib, lib.d3r_gemm_bf16(P, P, P, None, None, None, 128, 128, 64, 128, flag, None, None, 0, 0, 0, None), 'gemm')
        assert 'd3r_conv_transpose_bf16' in msg and 'd3r_conv3x3_head_tail' in msg, msg
