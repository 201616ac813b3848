"""The TMA-store epilogue of the 128x256 projection GEMMs (d3r_set_gemm_store(1), the default) against the register-store
epilogue (d3r_set_gemm_store(0)) and against torch.

The staged epilogue keeps the bias / GELU / RoPE arithmetic of the register path and only changes how the result reaches
global memory: a TMA store of bf16 tiles, or a TMA reduce-add into the fp32 residual stream.  Both must give the register
path's bits.  Every case runs on both kernel families, at the eight projection shapes of the forward with a partial last
tile, and at M where there are fewer tiles than CTAs or an odd number of M tiles per CTA pair."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from dust3r_b200 import _lib
from dust3r_b200._lib_fwd import F_BIAS, F_GELU, F_RELU, F_RESID_INPLACE, F_ROPE

# (N, K, epilogue) of the encoder (ViT-L) and decoder (ViT-B) projections: qkv, proj, fc1, fc2
PROJECTIONS = [(3072, 1024, 'rope'), (1024, 1024, 'resid'), (4096, 1024, 'gelu'), (1024, 4096, 'resid'),
               (2304, 768, 'rope'), (768, 768, 'resid'), (3072, 768, 'gelu'), (768, 3072, 'resid')]
CASES = ([(4100, N, K, epi) for N, K, epi in PROJECTIONS] +
         [(M, N, K, epi) for M in (1, 127, 130, 300) for N, K, epi in ((1024, 1024, 'gelu'), (2304, 768, 'rope'), (768, 3072, 'resid'))])
# token grid (gh, gw) of one image of M tokens, so that the RoPE oracle sees whole images
GRID = {4100: (41, 100), 1: (1, 1), 127: (1, 127), 130: (10, 13), 300: (12, 25)}


@pytest.fixture(params=[0, 1], ids=['cta1', 'cta_pair'], autouse=True)
def gemm_impl(request):
    lib = _lib.get_lib()
    lib.d3r_set_gemm_impl(request.param)
    yield request.param
    lib.d3r_set_gemm_impl(2)
    lib.d3r_set_gemm_store(1)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _rand(shape, dev, scale=1.0, seed=0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


def gemm(store, A, B, bias, flags, out, ldo, rope=None):
    """out: the first element of an [M, ldo] matrix of which the kernel writes the first N columns"""
    lib = _lib.get_lib()
    M, K = A.shape
    N = B.shape[0]
    cos, sin, rope_cols, tpi, gw = rope if rope is not None else (None, None, 0, 0, 0)
    lib.d3r_set_gemm_store(store)
    try:
        _lib.check(lib.d3r_gemm_bf16(_p(A), _p(B), C.c_void_p(out.data_ptr()), _p(bias), _p(None), _p(None), M, N, K, ldo, flags,
                                     _p(cos), _p(sin), rope_cols, tpi, gw, _lib.stream_ptr()))
    finally:
        lib.d3r_set_gemm_store(1)
    torch.cuda.synchronize()


def bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def assert_same_bits(a, b):
    assert torch.equal(bits(a), bits(b)), int((bits(a) != bits(b)).sum())


def residual_start(M, N, dev, seed):
    """mixed signs, exact zeros of both signs, tiny normal values and subnormals"""
    x = _rand((M, N), dev, seed=seed)
    g = torch.Generator(device='cpu').manual_seed(seed + 1)
    kind = torch.randint(0, 6, (M, N), generator=g).to(dev)
    x = torch.where(kind == 1, torch.zeros_like(x), x)
    x = torch.where(kind == 2, torch.full_like(x, -0.0), x)
    x = torch.where(kind == 3, x * 1e-31, x)
    x = torch.where(kind == 4, x * 1e-39, x)        # below the smallest normal fp32 (1.18e-38)
    return x


def operands(M, N, K, dev):
    A = _rand((M, K), dev, seed=41).bfloat16()
    A[::7] = 0                                        # zero rows and zero bias columns: the residual update adds a zero,
    B = _rand((N, K), dev, scale=K ** -0.5, seed=42).bfloat16()
    bias = _rand((N,), dev, seed=43)
    bias[::5] = 0                                     # and x + 0 must keep x's bits, subnormal x included
    return A, B, bias


def run_act(M, N, K, dev, ldo=None, offset=0):
    """bias + GELU, and ReLU without bias"""
    ldo = ldo or N
    A, B, bias = operands(M, N, K, dev)
    prod = A.float() @ B.float().T
    for b, flags, ref in ((bias, F_BIAS | F_GELU, torch.nn.functional.gelu(prod + bias)), (None, F_RELU, prod.relu())):
        outs = []
        for store in (0, 1):
            buf = torch.full((M * ldo + offset + 64,), 7.0, dtype=torch.bfloat16, device=dev)
            gemm(store, A, B, b, flags, buf[offset:], ldo)
            outs.append(buf)
        assert_same_bits(outs[0], outs[1])
        out = outs[1][offset:offset + M * ldo].view(M, ldo)
        assert (out[:, :N].float() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())
        assert (out[:, N:] == 7.0).all() and (outs[1][:offset] == 7.0).all() and (outs[1][offset + M * ldo:] == 7.0).all()


def run_resid(M, N, K, dev, ldo=None, offset=0):
    ldo = ldo or N
    A, B, bias = operands(M, N, K, dev)
    x0 = residual_start(M, ldo, dev, seed=44)
    guard = torch.full((8 * ldo + 64,), 7.0, device=dev)             # the rows after M must stay untouched
    bufs = []
    for store in (0, 1):
        buf = torch.cat((torch.full((offset,), 7.0, device=dev), x0.reshape(-1), guard))
        gemm(store, A, B, bias, F_BIAS | F_RESID_INPLACE, buf[offset:], ldo)   # twice on the same stream: the second
        gemm(store, A, B, None, F_RESID_INPLACE, buf[offset:], ldo)            # update adds onto the first
        bufs.append(buf)
    assert_same_bits(bufs[0], bufs[1])
    got = bufs[1][offset:offset + M * ldo].view(M, ldo)
    prod = A.float() @ B.float().T
    tol = 3e-4 * max(1.0, (K / 320) ** 0.5)
    assert (got[:, :N] - (x0[:, :N] + 2 * prod + bias)).abs().max().item() < 2 * tol
    assert_same_bits(got[:, N:], x0[:, N:])
    assert (bufs[1][:offset] == 7.0).all() and torch.equal(bufs[1][offset + M * ldo:], guard)


def run_rope(M, N, K, dev):
    from oracle.forward_oracle import rope2d, positions, rope_tables
    hd = 64
    Cdim = N // 3
    nh = Cdim // hd
    gh, gw = GRID[M]
    A, B, bias = operands(M, N, K, dev)
    cos, sin = rope_tables(hd, max(gh, gw), 100.0)
    cos, sin = cos.to(dev).contiguous(), sin.to(dev).contiguous()
    outs = []
    for store in (0, 1):
        out = torch.full((M, N), float('nan'), dtype=torch.bfloat16, device=dev)
        gemm(store, A, B, bias, F_BIAS | F_ROPE, out, N, rope=(cos, sin, 2 * Cdim, gh * gw, gw))
        outs.append(out)
    assert_same_bits(outs[0], outs[1])
    lin = (A.float() @ B.float().T + bias).cpu().reshape(1, M, 3, nh, hd).permute(2, 0, 3, 1, 4)
    pos = positions(1, gh, gw)
    ref = torch.stack((rope2d(lin[0], pos, 100.0), rope2d(lin[1], pos, 100.0), lin[2]), 0).permute(1, 3, 0, 2, 4).reshape(M, N)
    assert torch.isfinite(outs[1].float()).all()
    assert (outs[1].float().cpu() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())


@pytest.mark.timeout(300)
@pytest.mark.parametrize('M,N,K,epi', CASES)
def test_tma_store_matches_register_store(cuda_device, M, N, K, epi):
    {'gelu': run_act, 'resid': run_resid, 'rope': run_rope}[epi](M, N, K, cuda_device)


@pytest.mark.timeout(300)
@pytest.mark.parametrize('M,N,K', [(300, 1024, 1024), (4100, 768, 768)])
def test_tma_store_strided_output(cuda_device, M, N, K):
    """ldo > N with 16-byte rows takes the TMA path; a row stride or base that is not a multiple of 16 bytes takes the
    register stores; all agree bit for bit and leave the columns past N alone"""
    run_act(M, N, K, cuda_device, ldo=N + 64)
    run_act(M, N, K, cuda_device, ldo=N + 4)             # 8-byte aligned rows
    run_act(M, N, K, cuda_device, ldo=N, offset=2)       # 4-byte aligned base
    run_resid(M, N, K, cuda_device, ldo=N + 32)
    run_resid(M, N, K, cuda_device, ldo=N + 2)
    run_resid(M, N, K, cuda_device, ldo=N, offset=2)     # 8-byte aligned base
