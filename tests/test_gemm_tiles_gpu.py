"""The specialised bf16-output epilogues on the 128x256 tiles, through the C ABI, on both kernel families.

test_gemm_gpu.py checks RoPE with an fp32 output, which runs the generic epilogue; the forward stores q / k / v as
bf16, which runs the EPI_ROPE specialisation.  N % 256 == 0 here, so that specialisation runs on 128x256 tiles."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from dust3r_b200 import _lib
from dust3r_b200._lib_fwd import F_BIAS, F_GELU, F_ROPE


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def gemm(A, B, bias, flags, rope=None):
    """bf16 output, ldo = N; the output starts as NaN so that an element left unwritten fails the comparison"""
    M, K = A.shape
    N = B.shape[0]
    out = torch.full((M, N), float('nan'), dtype=torch.bfloat16, device=A.device)
    cos, sin, rope_cols, tpi, gw = rope if rope is not None else (None, None, 0, 0, 0)
    _lib.check(_lib.get_lib().d3r_gemm_bf16(_p(A), _p(B), _p(out), _p(bias), _p(None), _p(None), M, N, K, N, flags, _p(cos),
                                            _p(sin), rope_cols, tpi, gw, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out


def _rand(shape, dev, scale=1.0, seed=0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


@pytest.fixture(params=[0, 1], ids=['cta1', 'cta_pair'], autouse=True)
def gemm_impl(request):
    lib = _lib.get_lib()
    lib.d3r_set_gemm_impl(request.param)
    yield request.param
    lib.d3r_set_gemm_impl(2)


@pytest.mark.timeout(300)
@pytest.mark.parametrize('Bimg,gh,gw,kv', [pytest.param(3, 6, 10, False, id='3-6-10'), pytest.param(5, 12, 16, False, id='5-12-16'),
                                           pytest.param(3, 21, 32, True, id='kv-3-21-32'),
                                           pytest.param(3, 32, 21, False, id='portrait-3-32-21')])
def test_gemm_rope_bf16_matches_oracle(cuda_device, Bimg, gh, gw, kv):
    """QKV projection with fused 2D RoPE stored as bf16 == oracle rope2d(linear) (croco/models/pos_embed.py:113-157).
    kv: the decoder's fused k|v projection of the cross attention, rope_cols = N / 2: k rotated, v left as it is.  The
    portrait grid (gh > gw) has row positions past gw."""
    from oracle.forward_oracle import rope2d, positions, rope_tables
    nh, hd = 4, 64
    Cdim = nh * hd
    Ntok = gh * gw
    M = Bimg * Ntok
    parts = 2 if kv else 3
    x = _rand((M, Cdim), cuda_device, seed=31).bfloat16()
    Wqkv = _rand((parts * Cdim, Cdim), cuda_device, scale=Cdim ** -0.5, seed=32).bfloat16()
    bias = _rand((parts * Cdim,), cuda_device, seed=33)
    cos, sin = rope_tables(hd, max(gh, gw), 100.0)
    cos, sin = cos.to(cuda_device).contiguous(), sin.to(cuda_device).contiguous()
    out = gemm(x, Wqkv, bias, F_BIAS | F_ROPE, rope=(cos, sin, (parts - 1) * Cdim, Ntok, gw))
    lin = (x.float() @ Wqkv.float().T + bias).cpu().reshape(Bimg, Ntok, parts, nh, hd).permute(2, 0, 3, 1, 4)
    pos = positions(Bimg, gh, gw)
    rotated = [rope2d(lin[i], pos, 100.0) for i in range(parts - 1)]
    ref = torch.stack(rotated + [lin[parts - 1]], 0).permute(1, 3, 0, 2, 4).reshape(M, parts * Cdim)
    assert torch.isfinite(out.float()).all()
    assert (out.float().cpu() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())
    if kv:
        # v is the plain projection: within one bf16 rounding of it, never rotated
        v = lin[1].permute(0, 2, 1, 3).reshape(M, Cdim)
        assert ((out.float().cpu()[:, Cdim:] - v).abs() <= 2.0 ** -8 * v.abs() + 1e-3).all()


@pytest.mark.timeout(300)
@pytest.mark.parametrize('M,N,K', [(300, 256, 64), (1000, 1536, 768), (4100, 4096, 1024)])
def test_gemm_gelu_bf16_wide_tiles(cuda_device, M, N, K):
    """bias + GELU -> bf16 on 128x256 tiles: partial last M tile, single and many k-blocks."""
    A = _rand((M, K), cuda_device, seed=34).bfloat16()
    B = _rand((N, K), cuda_device, scale=K ** -0.5, seed=35).bfloat16()
    bias = _rand((N,), cuda_device, seed=36)
    ref = torch.nn.functional.gelu(A.float() @ B.float().T + bias)
    out = gemm(A, B, bias, F_BIAS | F_GELU)
    assert torch.isfinite(out.float()).all()
    assert (out.float() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())
