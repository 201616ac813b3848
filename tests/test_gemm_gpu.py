"""wgmma GEMM / implicit-GEMM conv kernels through the C ABI vs plain torch fp32 on the same
bf16-rounded operands.  Tolerance: the kernel accumulates in fp32 (registers) exactly like the torch
reference up to summation order; outputs stored as bf16 carry one rounding (rel 2^-8)."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from dust3r_b200 import _lib
from dust3r_b200._lib_fwd import (F_BIAS, F_GELU, F_RELU, F_OUT_F32, F_RESID_INPLACE, F_ADD0, F_ADD1, F_OUT2_RELU,
                                  F_ROPE, F_OUT2_BF16)


@pytest.fixture(params=[0, 1], ids=['cta1', 'cta_pair'], autouse=True)
def gemm_impl(request):
    """every test runs on both kernel families: 1-CTA and CTA-pair (a cluster of two sharing a multicast B tile)"""
    lib = _lib.get_lib()
    lib.d3r_set_gemm_impl(request.param)
    yield request.param
    lib.d3r_set_gemm_impl(2)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def gemm(A, B, bias=None, flags=0, out_dtype=torch.bfloat16, out=None, add0=None, out2=None, rope=None):
    lib = _lib.get_lib()
    M, K = A.shape
    N = B.shape[0]
    if out is None:
        out = torch.full((M, N), float('nan'), dtype=out_dtype, device=A.device)
    cos = sin = None
    rope_cols = tpi = gw = 0
    if rope is not None:
        cos, sin, rope_cols, tpi, gw = rope
    _lib.check(lib.d3r_gemm_bf16(_p(A), _p(B), _p(out), _p(bias), _p(add0), _p(out2), M, N, K, N, flags, _p(cos), _p(sin),
                                 rope_cols, tpi, gw, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out


def _rand(shape, dev, scale=1.0, seed=0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


@pytest.mark.timeout(300)
@pytest.mark.parametrize('M,N,K', [(128, 256, 64), (300, 256, 192), (128, 64, 96), (257, 96, 1024), (4096, 3072, 1024),
                                   (1000, 768, 4096), (2048, 192, 768), (640, 128, 256), (333, 2304, 768)])
def test_gemm_bias_bf16(cuda_device, M, N, K):
    A = _rand((M, K), cuda_device, seed=1).bfloat16()
    B = _rand((N, K), cuda_device, scale=K ** -0.5, seed=2).bfloat16()
    bias = _rand((N,), cuda_device, seed=3)
    ref = A.float() @ B.float().T + bias
    out = gemm(A, B, bias, F_BIAS)
    err = (out.float() - ref).abs().max().item()
    assert torch.isfinite(out.float()).all()
    assert err <= 2e-2 * max(1.0, ref.abs().max().item()), err
    out32 = gemm(A, B, bias, F_BIAS | F_OUT_F32, out_dtype=torch.float32)
    assert (out32 - ref).abs().max().item() <= 2e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.timeout(300)
def test_gemm_epilogues(cuda_device):
    M, N, K = 777, 512, 320
    A = _rand((M, K), cuda_device, seed=4).bfloat16()
    B = _rand((N, K), cuda_device, scale=K ** -0.5, seed=5).bfloat16()
    bias = _rand((N,), cuda_device, seed=6)
    lin = A.float() @ B.float().T + bias
    # GELU (erf)
    out = gemm(A, B, bias, F_BIAS | F_GELU | F_OUT_F32, out_dtype=torch.float32)
    assert (out - torch.nn.functional.gelu(lin)).abs().max().item() < 3e-4
    # in-place fp32 residual + bf16 copy
    resid = _rand((M, N), cuda_device, seed=7)
    buf = resid.clone()
    copy = torch.zeros((M, N), dtype=torch.bfloat16, device=cuda_device)
    gemm(A, B, bias, F_BIAS | F_RESID_INPLACE | F_OUT2_BF16, out=buf, out2=copy)
    assert (buf - (resid + lin)).abs().max().item() < 3e-4
    assert (copy.float() - (resid + lin)).abs().max().item() < 4e-2
    # bf16 addend + relu + dual relu output
    add = _rand((M, N), cuda_device, seed=8).bfloat16()
    out2 = torch.zeros((M, N), dtype=torch.bfloat16, device=cuda_device)
    out = gemm(A, B, bias, F_BIAS | F_ADD0 | F_OUT2_RELU, add0=add, out2=out2)
    ref = lin + add.float()
    assert (out.float() - ref).abs().max().item() < 4e-2
    assert (out2.float() - ref.relu()).abs().max().item() < 4e-2
    # no bias, relu
    out = gemm(A, B, None, F_RELU | F_OUT_F32, out_dtype=torch.float32)
    assert (out - (A.float() @ B.float().T).relu()).abs().max().item() < 3e-4


@pytest.mark.timeout(300)
@pytest.mark.parametrize('M,N,K', [(777, 512, 320), (1000, 768, 1024), (130, 256, 64), (4100, 1024, 4096)])
def test_gemm_specialised_epilogues(cuda_device, M, N, K):
    """The compile-time epilogue specialisations (N % 128 == 0): in-place residual update (rows past M
    are left untouched), bias/GELU -> bf16, bias/ReLU -> bf16, with and without bias."""
    A = _rand((M, K), cuda_device, seed=21).bfloat16()
    B = _rand((N, K), cuda_device, scale=K ** -0.5, seed=22).bfloat16()
    bias = _rand((N,), cuda_device, seed=23)
    prod = A.float() @ B.float().T
    tol = 3e-4 * max(1.0, (K / 320) ** 0.5)
    # EPI_RESID: twice onto the same stream (the second update sees the first)
    resid = _rand((M, N), cuda_device, seed=24)
    guard = torch.full((8, N), 7.0, device=cuda_device)            # rows right behind the matrix must stay untouched
    buf = torch.cat((resid, guard))
    gemm(A, B, bias, F_BIAS | F_RESID_INPLACE, out=buf[:M])
    assert (buf[:M] - (resid + prod + bias)).abs().max().item() < tol
    gemm(A, B, None, F_RESID_INPLACE, out=buf[:M])
    assert (buf[:M] - (resid + 2 * prod + bias)).abs().max().item() < 2 * tol
    assert torch.equal(buf[M:], guard)
    # EPI_ACT
    out = gemm(A, B, bias, F_BIAS | F_GELU)
    ref = torch.nn.functional.gelu(prod + bias)
    assert (out.float() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())
    out = gemm(A, B, None, F_RELU)
    assert (out.float() - prod.relu()).abs().max().item() <= 2e-2 * max(1.0, prod.abs().max().item())


@pytest.mark.timeout(300)
def test_gemm_rope_matches_oracle(cuda_device):
    """QKV projection with fused 2D RoPE == oracle rope2d(linear) (croco/models/pos_embed.py:113-157)."""
    from oracle.forward_oracle import rope2d, positions, rope_tables
    Bimg, gh, gw, nh, hd = 3, 6, 10, 4, 64
    Cdim = nh * hd
    Ntok = gh * gw
    M = Bimg * Ntok
    x = _rand((M, Cdim), cuda_device, seed=9).bfloat16()
    Wqkv = _rand((3 * Cdim, Cdim), cuda_device, scale=Cdim ** -0.5, seed=10).bfloat16()
    bias = _rand((3 * Cdim,), cuda_device, seed=11)
    cos, sin = rope_tables(hd, max(gh, gw), 100.0)
    cos, sin = cos.to(cuda_device).contiguous(), sin.to(cuda_device).contiguous()
    out = gemm(x, Wqkv, bias, F_BIAS | F_ROPE | F_OUT_F32, out_dtype=torch.float32, rope=(cos, sin, 2 * Cdim, Ntok, gw))
    lin = (x.float() @ Wqkv.float().T + bias).cpu().reshape(Bimg, Ntok, 3, nh, hd).permute(2, 0, 3, 1, 4)
    pos = positions(Bimg, gh, gw)
    q = rope2d(lin[0], pos, 100.0)
    k = rope2d(lin[1], pos, 100.0)
    ref = torch.stack((q, k, lin[2]), 0).permute(1, 3, 0, 2, 4).reshape(M, 3 * Cdim)
    assert (out.cpu() - ref).abs().max().item() < 5e-4


def conv(x, w, bias=None, flags=0, add0=None, add1=None, out2=None):
    lib = _lib.get_lib()
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    wp = w.permute(0, 2, 3, 1).contiguous().bfloat16()     # [Cout][ky][kx][Cin]
    out = torch.full((B, H, W, Cout), float('nan'), dtype=torch.bfloat16, device=x.device)
    _lib.check(lib.d3r_conv3x3_bf16(_p(x), _p(wp), _p(out), _p(bias), _p(add0), _p(add1), _p(out2), B, H, W, Cin, Cout, flags,
                                    _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out


@pytest.mark.timeout(300)
@pytest.mark.parametrize('B,H,W,Cin,Cout', [(2, 24, 32, 96, 256), (1, 12, 16, 768, 256), (2, 48, 64, 256, 256),
                                            (1, 96, 128, 256, 128), (3, 10, 14, 192, 256), (1, 20, 200, 128, 128)])
def test_conv3x3_matches_torch(cuda_device, B, H, W, Cin, Cout):
    x = _rand((B, H, W, Cin), cuda_device, seed=12).bfloat16()
    w = _rand((Cout, Cin, 3, 3), cuda_device, scale=(9 * Cin) ** -0.5, seed=13).bfloat16()
    bias = _rand((Cout,), cuda_device, seed=14)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1)
    out = conv(x, w, bias, F_BIAS)
    assert torch.isfinite(out.float()).all()
    assert (out.float() - ref).abs().max().item() < 4e-2
    add0 = _rand((B, H, W, Cout), cuda_device, seed=15).bfloat16()
    add1 = _rand((B, H, W, Cout), cuda_device, seed=16).bfloat16()
    out2 = torch.zeros_like(out)
    out = conv(x, w, bias, F_BIAS | F_ADD0 | F_ADD1 | F_OUT2_RELU, add0=add0, add1=add1, out2=out2)
    ref2 = ref + add0.float() + add1.float()
    assert (out.float() - ref2).abs().max().item() < 6e-2
    assert (out2.float() - ref2.relu()).abs().max().item() < 6e-2
