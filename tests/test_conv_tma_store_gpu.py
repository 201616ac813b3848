"""The staged TMA epilogue of the DPT 3x3 convolutions (d3r_set_conv_store(1), the default: conv_kernel on 128x256 or
128x128 tiles) against the register-store kernels on 128x128 tiles (d3r_set_conv_store(0)), bit for bit, on both kernel
families; each case also against torch conv2d on the same bf16 operands; and the vitl_512_dpt forward under both settings.

The two paths round the same fp32 values in the same order (acc + bias, + add0, + add1, ReLU; out2 = relu of that), so
they must agree in every bit.  Outputs start as NaN and are followed by one pixel row of guard elements that must keep
their value: ragged x / y tiles and the missing M tile of an odd count are clipped by the tensor maps, not written."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from dust3r_b200 import _lib
from dust3r_b200._lib_fwd import F_BIAS, F_RELU, F_ADD0, F_ADD1, F_OUT2_RELU
from test_forward_ops_gpu import _p, _call, _randn, _nan_buffer, _guard_ok, gemm_family  # noqa: F401  (fixture)
from test_gemm_conv_float64_gpu import CONV_TABLE

BF16 = torch.bfloat16
RCU2 = F_BIAS | F_ADD0 | F_ADD1 | F_OUT2_RELU
# Cases the (B = 2) float64 tables do not reach: an odd number of M tiles (3 images of one 8x16 tile; 7 tiles of 2x64
# with ragged x and y), and launches with >= 4 waves of CTA-pair items, which take the 128x256 tiles: level 0 of the
# 24x32 grid at B = 6, the portrait level 0 (W = 84, ragged x) at B = 5, and 603 tiles of 1x128 (odd, ragged x).
EXTRA = [
    ('odd_tiles', 256, 256, RCU2, [(3, 7, 7), (1, 13, 40)]),
    ('odd_tiles_conv1', 256, 256, F_BIAS | F_RELU, [(3, 7, 7), (1, 13, 40)]),
    ('wide_rcu1_conv2', 256, 256, RCU2, [(6, 96, 128), (5, 128, 84), (3, 201, 84)]),
    ('wide_rcu2_conv2', 256, 256, F_BIAS | F_ADD0, [(6, 96, 128), (3, 201, 84)]),
    ('wide_rcu_conv1', 256, 256, F_BIAS | F_RELU, [(6, 96, 128), (3, 201, 84)]),
    ('wide_layer_rn0', 96, 256, F_OUT2_RELU, [(6, 96, 128)]),
    ('wide_head0', 256, 128, F_BIAS, [(6, 96, 128)]),
]
CASES = [(name, Cin, Cout, fl, c) for name, Cin, Cout, fl, cases in CONV_TABLE + EXTRA for c in cases]


def _bits(t):
    return t.view(torch.int16)


@pytest.fixture
def conv_store_restored():
    lib = _lib.get_lib()
    try:
        yield lib
    finally:
        lib.d3r_set_conv_store(1)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('case', CASES, ids=[f'{c[0]}-{c[4][0]}x{c[4][1]}x{c[4][2]}' for c in CASES])
def test_conv_store_bit_identical(cuda_device, gemm_family, conv_store_restored, case):
    dev = cuda_device
    lib = conv_store_restored
    name, Cin, Cout, flags, (B, H, W) = case
    seed = 31000 + 17 * CASES.index(case)
    x = _randn((B, H, W, Cin), seed, dev).to(BF16)
    w = _randn((Cout, Cin, 3, 3), seed + 1, dev, scale=(9 * Cin) ** -0.5).to(BF16)
    wp = w.permute(0, 2, 3, 1).contiguous()
    bias = _randn((Cout,), seed + 2, dev).float() if flags & F_BIAS else None
    add0 = _randn((B, H, W, Cout), seed + 3, dev).to(BF16) if flags & F_ADD0 else None
    add1 = _randn((B, H, W, Cout), seed + 4, dev).to(BF16) if flags & F_ADD1 else None
    n = B * H * W * Cout
    res = {}
    for store in (0, 1):
        lib.d3r_set_conv_store(store)
        o = _nan_buffer(n, BF16, dev, guard=W * Cout)[0]
        o2 = _nan_buffer(n, BF16, dev, guard=W * Cout)[0] if flags & F_OUT2_RELU else None
        _call(lib.d3r_conv3x3_bf16(_p(x), _p(wp), _p(o), _p(bias), _p(add0), _p(add1), _p(o2), B, H, W, Cin, Cout, flags,
                                   _lib.stream_ptr()))
        res[store] = (o, o2)
    what = f'{name} impl={gemm_family} B={B} {H}x{W} Cin={Cin} Cout={Cout}'
    for i, label in ((0, 'out'), (1, 'out2')):
        a, b = res[0][i], res[1][i]
        if a is None:
            continue
        assert _guard_ok(b, n), f'{what}: {label} guard written by the staged epilogue'
        assert torch.isfinite(b[:n].float()).all(), f'{what}: {label} has unwritten elements'
        diff = int((_bits(a) != _bits(b)).sum())
        assert diff == 0, f'{what}: {label}: {diff} elements differ between conv_store 0 and 1'
    # torch conv2d on the same bf16 operands (fp32, no TF32), the epilogue in fp32
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), padding=1).permute(0, 2, 3, 1)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    if bias is not None:
        ref = ref + bias
    for a in (add0, add1):
        if a is not None:
            ref = ref + a.float()
    if flags & F_RELU:
        ref = ref.clamp(min=0)
    out = res[1][0][:n].view(B, H, W, Cout).float()
    torch.testing.assert_close(out, ref, rtol=2.0 ** -7, atol=1e-2, msg=lambda m: f'{what} vs torch conv2d: {m}')
    if flags & F_OUT2_RELU:
        torch.testing.assert_close(res[1][1][:n].view(B, H, W, Cout).float(), ref.clamp(min=0), rtol=2.0 ** -7, atol=1e-2,
                                   msg=lambda m: f'{what} out2 vs torch conv2d: {m}')


@pytest.mark.timeout(1200)
def test_forward_same_bits_under_both_conv_stores(cuda_device, conv_store_restored):
    """vitl_512_dpt at 512x384, B = 2 pairs: pts3d and conf of both views equal bit for bit under conv_store 0 and 1"""
    from dust3r_b200.config import vitl_512_dpt
    from dust3r_b200.utils.synth import synth_images
    from test_forward_gpu import _build
    dev = cuda_device
    lib = conv_store_restored
    net, _ = _build(vitl_512_dpt(), 0, dev)
    packed = net.repack()
    imgs = torch.cat([im['img'] for im in synth_images(4, 384, 512, seed=3)]).to(dev)
    res = {}
    for store in (0, 1):
        lib.d3r_set_conv_store(store)
        r1, r2 = packed.forward(imgs, np.arange(2, dtype=np.int32), 2 + np.arange(2, dtype=np.int32), 2, 384, 512)
        torch.cuda.synchronize()
        res[store] = [t.clone() for t in (r1['pts3d'], r1['conf'], r2['pts3d'], r2['conf'])]
    for k, a, b in zip(('pts1', 'conf1', 'pts2', 'conf2'), res[0], res[1]):
        assert torch.isfinite(a).all(), k
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f'{k}: {int((a != b).sum())} elements differ'
