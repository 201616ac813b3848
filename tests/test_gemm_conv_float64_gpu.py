"""The projection GEMMs and the DPT 3x3 convolutions (gemm_kernel as a plain GEMM, mode 0, and as an implicit-GEMM 3x3
convolution, mode 1) against float64 torch on the same bf16 operands, element by element, at every (N, K, flags) the
forward calls them with; the 1-CTA and CTA-pair kernels, and the register-store and TMA-store epilogues, bit for bit; the
tables tied to the forward's actual launches; and the forward with programmatic dependent launch against the one without.

Notation and the bf16 output rule (U, g(K), |out - ref| <= U (|ref| + e) + e, >= 99 % exactly bf16(ref)) are those of
test_forward_ops_gpu.py, whose helpers this file uses.  The epilogue's own error terms, added to g(K) S (S = |A| |B|^T +
|bias|, K = 9 Cin for the convolutions), are derived in _epilogue64.  Every output and out2 starts as NaN and is followed by
guard elements (one row / one pixel row past M) that must keep their value; every check also builds references perturbed
by named small bugs and asserts that its bound rejects them.  Worst |err| / bound per case is printed (pytest -s or -rP)."""
import math
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from dust3r_b200 import _lib
from dust3r_b200._lib_fwd import (F_BIAS, F_GELU, F_RELU, F_OUT_F32, F_RESID_INPLACE, F_ADD0, F_ADD1, F_OUT2_RELU, F_ROPE,
                                  F_OUT2_BF16)
from test_forward_ops_gpu import (F64, GUARD, _p, _call, _gamma, _randn, _nan_buffer, _guard_ok, _check_bf16, _violations,
                                  gemm_family)  # noqa: F401  (gemm_family is a fixture)
from test_gemm_tma_store_gpu import residual_start

F_CONVT, F_HEAD_FINAL = 1 << 9, 1 << 10          # tested in test_forward_ops_gpu.py, not here
BF16 = torch.bfloat16


def _levels(gh, gw):
    """the four DPT pyramid levels of a token grid (run_dpt: Hs = {4gh, 2gh, gh, (gh-1)/2+1}, same for W)"""
    return [(4 * gh, 4 * gw), (2 * gh, 2 * gw), (gh, gw), ((gh - 1) // 2 + 1, (gw - 1) // 2 + 1)]


# ---- case tables (forward.cu) ------------------------------------------------------------------------------------------
# M cases (B, gh, gw), M = B gh gw; RoPE positions are (tok / gw, tok % gw) of tok = row % (gh gw)
TOKENS = [(2, 24, 32),     # 1536 rows: 12 whole M tiles
          (2, 21, 32),     # 1344: 11 M tiles, the second CTA of the last pair has no tile
          (1, 14, 14),     # 196: fewer work items than SMs
          (3, 32, 21),     # 2016: portrait grid, ragged last M tile
          (2, 7, 7),       # 98 < 128: one partial M tile
          (16, 24, 32)]    # 12288: several persistent rounds per CTA
H3 = [(2, 12, 16), (2, 11, 16), (2, 7, 7), (3, 16, 11), (16, 12, 16)]   # act3_down: M = B h3 w3 (24x32, 21x32, 14x14, 32x21)
LEVELS = [(2,) + _levels(24, 32)[0], (2,) + _levels(21, 32)[1], (3,) + _levels(32, 21)[2], (2,) + _levels(14, 14)[3]]
ABI = [(1, 10, 10), (3, 13, 20), (2, 41, 50)]

# (name, N, K, flags, rope_cols, M cases).  Encoder E = 1024 (MLP 4096), decoder D = 768 (MLP 3072).
GEMM_FORWARD = [
    ('enc_patch_embed', 1024, 768, F_BIAS | F_OUT_F32, 0, TOKENS),        # run_encoder: patch_embed -> x (fp32)
    ('enc_qkv', 3072, 1024, F_BIAS | F_ROPE, 2048, TOKENS),               # enc block qkv, q and k rotated
    ('enc_proj', 1024, 1024, F_BIAS | F_RESID_INPLACE, 0, TOKENS),        # enc block proj, x += ...
    ('enc_fc1', 4096, 1024, F_BIAS | F_GELU, 0, TOKENS),                  # enc block fc1
    ('enc_fc2', 1024, 4096, F_BIAS | F_RESID_INPLACE, 0, TOKENS),         # enc block fc2, x += ...
    ('dec_embed', 768, 1024, F_BIAS | F_OUT_F32, 0, TOKENS),              # decode_heads: decoder_embed -> x (fp32)
    ('dec_qkv', 2304, 768, F_BIAS | F_ROPE, 1536, TOKENS),                # dec_block qkv
    ('dec_proj', 768, 768, F_BIAS | F_RESID_INPLACE, 0, TOKENS),          # dec_block proj and cproj
    ('dec_projq', 768, 768, F_BIAS | F_ROPE, 768, TOKENS),                # dec_block projq: q rotated
    ('dec_projkv', 1536, 768, F_BIAS | F_ROPE, 768, TOKENS + [(3, 32, 24)]),  # dec_block projkv: k rotated at the memory
                                                                          # view's positions (21x32 for 24x32 queries), v not
    ('dec_fc1', 3072, 768, F_BIAS | F_GELU, 0, TOKENS),                   # dec_block fc1
    ('dec_fc2', 768, 3072, F_BIAS | F_RESID_INPLACE, 0, TOKENS),          # dec_block fc2
    ('linear_head', 1024, 768, F_BIAS | F_OUT_F32, 0, TOKENS),            # linear head (nch 4 x 16 x 16) -> fp32
    ('dpt_act_conv0', 96, 1024, F_BIAS, 0, TOKENS),                       # run_dpt act_conv[0]: one and a half 64-wide tiles
    ('dpt_act_conv1', 192, 768, F_BIAS, 0, TOKENS),                       # act_conv[1]
    ('dpt_act_conv2', 384, 768, F_BIAS, 0, TOKENS),                       # act_conv[2]: EPI_ACT on 128-wide tiles
    ('dpt_act_conv3', 768, 768, F_BIAS, 0, TOKENS),                       # act_conv[3]: EPI_ACT on 256-wide tiles
    ('dpt_act3_down', 768, 6912, F_BIAS, 0, H3),                          # act3_down on the 3x3 s2 im2col
    ('dpt_out_conv', 256, 256, F_BIAS, 0, LEVELS),                        # refinenet out_conv at every level
]
# reachable through d3r_gemm_bf16, not used by the forward: every gemm_kernel instantiation dispatch() can launch
GEMM_ABI = [
    ('abi_resid_n384', 384, 768, F_BIAS | F_RESID_INPLACE, 0, ABI),       # EPI_RESID on 128-wide tiles
    ('abi_rope_n384', 384, 256, F_BIAS | F_ROPE, 256, ABI),               # EPI_ROPE on 128-wide tiles
    ('abi_gelu_n640', 640, 320, F_BIAS | F_GELU, 0, ABI),                 # EPI_ACT GELU on 128-wide tiles
    ('abi_relu_n1024', 1024, 320, F_RELU, 0, ABI),                        # EPI_ACT ReLU without bias, 256-wide tiles
    ('abi_n32', 32, 256, F_BIAS | F_RELU, 0, ABI),                        # one half-empty 64-wide tile
    ('abi_n160', 160, 512, F_BIAS, 0, ABI),                               # EPI_ACT, second 128-wide tile 32 columns
    ('abi_add0_out2relu', 512, 320, F_BIAS | F_ADD0 | F_OUT2_RELU, 0, ABI),            # generic epilogue, mode 0
    ('abi_resid_out2bf16', 768, 768, F_BIAS | F_RESID_INPLACE | F_OUT2_BF16, 0, ABI),  # generic: fp32 += and a bf16 copy
    ('abi_gelu_f32', 256, 64, F_BIAS | F_GELU | F_OUT_F32, 0, ABI),       # generic GELU -> fp32, short K
]
GEMM_TABLE = GEMM_FORWARD + GEMM_ABI

# (name, Cin, Cout, flags, (B, H, W) cases); F = 256.  Levels of the 24x32, portrait 32x21 and 14x14 grids give every
# tile_w the host picks (W 128 / 84 -> 128, 64 / 42 / 56 -> 64, 32 / 21 / 28 -> 32, 16 / 11 / 14 / 7 -> 16), ragged x
# tiles (84, 42, 21, 11, 7) and ragged y tiles (H 12 and 14 / 7 in tiles of 8 rows).
CONV_GRIDS = [(24, 32), (32, 21), (14, 14)]
ALL_LEVELS = [(2,) + lv for g in CONV_GRIDS for lv in _levels(*g)]
CONV_FORWARD = [
    ('layer_rn0', 96, 256, F_OUT2_RELU, [(2,) + _levels(*g)[0] for g in CONV_GRIDS]),   # layer_rn[k]: raw + relu copy
    ('layer_rn1', 192, 256, F_OUT2_RELU, [(2,) + _levels(*g)[1] for g in CONV_GRIDS]),
    ('layer_rn2', 384, 256, F_OUT2_RELU, [(2,) + _levels(*g)[2] for g in CONV_GRIDS]),
    ('layer_rn3', 768, 256, F_OUT2_RELU, [(2,) + _levels(*g)[3] for g in CONV_GRIDS]),
    ('rcu_conv1', 256, 256, F_BIAS | F_RELU, ALL_LEVELS),                               # rcu1_conv1 and rcu2_conv1
    ('rcu1_conv2', 256, 256, F_BIAS | F_ADD0 | F_ADD1 | F_OUT2_RELU, ALL_LEVELS),       # + r[lvl] + path, relu copy
    ('rcu2_conv2', 256, 256, F_BIAS | F_ADD0, ALL_LEVELS),                              # + the fusion sum
    ('head0', 256, 128, F_BIAS, [(2, 192, 256), (2, 256, 168)]),                        # 8gh x 8gw: two x tiles per row
]
CONV_ABI = [
    ('abi_cin8', 8, 256, F_BIAS | F_RELU, [(2, 20, 30), (3, 5, 130)]),                 # Cin < one 64-channel block
    ('abi_cout96', 256, 96, F_BIAS | F_ADD0 | F_ADD1 | F_OUT2_RELU, [(2, 9, 40)]),      # 64-wide tiles, ragged N
]
CONV_TABLE = CONV_FORWARD + CONV_ABI

# every gemm_kernel<BLOCK_N, EPI, PAIR, TMA_STORE> dispatch() launches, as (profiler tag, epilogue, store setting): the
# store setting only selects a different kernel for the specialised epilogues on 256-wide tiles
INSTANTIATIONS = ({(f'gemm_wgmma{p}_bn256', epi, store) for p in ('', '_2cta') for epi in (1, 2, 3) for store in (0, 1)} |
                  {(f'gemm_wgmma{p}_bn128', epi, None) for p in ('', '_2cta') for epi in (0, 1, 2, 3)} |
                  {('gemm_wgmma_bn64', 0, None), ('conv3x3_wgmma', 0, None), ('conv3x3_wgmma_2cta', 0, None)})


def _table_keys():
    """(N, K, flags, mode) of every table row, as the profiler records a launch"""
    return ({(N, K, fl, 0) for _, N, K, fl, _, _ in GEMM_TABLE} |
            {(Cout, 9 * Cin, fl, 1) for _, Cin, Cout, fl, _ in CONV_TABLE})


# ---- float64 reference of the epilogue -------------------------------------------------------------------------------
def _rope_tables(dev):
    """the forward's tables (model.py): angle[p][k] = p * 100^(-k/16) in fp32, cos / sin in fp32, 64 positions"""
    inv_freq = 1.0 / (100.0 ** (torch.arange(0, 16).float() / 16))
    ang = torch.arange(64).float()[:, None] * inv_freq[None, :]
    return ang.cos().to(dev).contiguous(), ang.sin().to(dev).contiguous()


def _rope64(y, e, rope, swap_yx=False):
    """2D RoPE of the columns < rope_cols: every 32-column chunk is the y (even chunk) or x (odd chunk) half of a 64-wide
    head, pairs (k, k + 16) rotated by the angle of position pos: u' = u c - w s, w' = w c + u s.  The kernel rounds
    twice per output in fp32 (a product and an FMA) on top of the input errors:  e' = |c| e_u + |s| e_w + 2^-22 (|uc| + |ws|)."""
    cos, sin, rope_cols, tpi, gw = rope
    M = y.shape[0]
    tok = torch.arange(M, device=y.device) % tpi
    py, px = tok // gw, tok % gw
    if swap_yx:
        py, px = px, py
    nch = rope_cols // 32
    even = (torch.arange(nch, device=y.device) % 2 == 0).view(1, nch, 1)
    c = torch.where(even, cos.double()[py][:, None], cos.double()[px][:, None])       # (M, nch, 16)
    s = torch.where(even, sin.double()[py][:, None], sin.double()[px][:, None])
    y, e = y.clone(), e.clone()
    yv, ev = y[:, :rope_cols].view(M, nch, 2, 16), e[:, :rope_cols].view(M, nch, 2, 16)
    u, w, eu, ew = yv[:, :, 0].clone(), yv[:, :, 1].clone(), ev[:, :, 0].clone(), ev[:, :, 1].clone()
    yv[:, :, 0], yv[:, :, 1] = u * c - w * s, w * c + u * s
    ev[:, :, 0] = c.abs() * eu + s.abs() * ew + 2.0 ** -22 * ((u * c).abs() + (w * s).abs())
    ev[:, :, 1] = c.abs() * ew + s.abs() * eu + 2.0 ** -22 * ((w * c).abs() + (u * s).abs())
    return y, e


def _gelu64(y, kind='erf'):
    if kind == 'tanh':
        return 0.5 * y * (1 + torch.tanh(math.sqrt(2 / math.pi) * (y + 0.044715 * y ** 3)))
    return 0.5 * y * (1 + torch.erf(y / math.sqrt(2)))


def _epilogue64(P, S, K, flags, bias=None, add0=None, add1=None, rope=None, resid=None, gelu='erf', swap_yx=False):
    """Float64 value of the kernel's result from the exact product P = A B^T (S = |A| |B|^T), in the kernel's order
    (bias, GELU, RoPE, addends, ReLU, residual), and e, a bound on |fp32 result - value| before the final bf16 rounding:
      accumulation and bias:  e = g(K) (S + |bias|);
      GELU (gelu_erf):  |gelu'| <= 1.13, so e -> 1.13 e, plus the A&S 7.1.26 erfc error 1.5e-7 scaled by |y| / 2, a relative
        2^-19 (1 + y^2) of the tail h = y/2 erfc(|y|/sqrt2) for rcp.approx / ex2.approx / the fp32 polynomial and the
        rounding of the argument u^2 of ex2, and 2^-23 |gelu| for the final subtraction;
      RoPE: _rope64;
      each fp32 addition (addends, residual): e -> e (1 + 2^-22) + 2^-23 |sum|.
    """
    y = P.clone()
    Sb = S
    if flags & F_BIAS:
        y += bias
        Sb = S + bias.abs()
    e = _gamma(K) * Sb
    if flags & F_GELU:
        y0 = y
        y = _gelu64(y0, gelu)
        h = 0.5 * y0.abs() * torch.special.erfc(y0.abs() / math.sqrt(2))
        e = 1.13 * e + 1e-7 * y0.abs() + 2.0 ** -19 * h * (1 + y0 * y0) + 2.0 ** -23 * y.abs()
    if flags & F_ROPE:
        y, e = _rope64(y, e, rope, swap_yx)
    for fl, a in ((F_ADD0, add0), (F_ADD1, add1)):
        if flags & fl and a is not None:
            y = y + a
            e = e * (1 + 2.0 ** -22) + 2.0 ** -23 * y.abs()
    if flags & F_RELU:
        y = y.clamp(min=0)
    if flags & F_RESID_INPLACE:
        y = resid + y
        e = e * (1 + 2.0 ** -22) + 2.0 ** -23 * y.abs()
    return y, e


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32)


def _fp32_ratio(out, ref, e):
    return ((out.double() - ref).abs() / (e + 1e-30)).max().item()


# ---- the plain GEMM (mode 0) -------------------------------------------------------------------------------------------
def _gemm_operands(row_i, case_i, N, K, flags, B, gh, gw, dev):
    M = B * gh * gw
    seed = 7000 + 100 * row_i + 10 * case_i
    ops = dict(M=M, A=_randn((M, K), seed, dev).to(BF16), W=_randn((N, K), seed + 1, dev, scale=K ** -0.5).to(BF16))
    ops['bias'] = _randn((N,), seed + 2, dev).float() if flags & F_BIAS else None
    ops['add0'] = _randn((M, N), seed + 3, dev).to(BF16) if flags & F_ADD0 else None
    ops['resid'] = residual_start(M, N, dev, seed + 4) if flags & F_RESID_INPLACE else None
    return ops


def _run_gemm(lib, ops, N, K, flags, rope, dev):
    """one d3r_gemm_bf16 call; returns (out buffer, out2 buffer or None), each M x N elements then one guard row"""
    M = ops['M']
    n = M * N
    if flags & F_RESID_INPLACE:
        buf = torch.cat((ops['resid'].reshape(-1), torch.full((N,), GUARD, device=dev)))
    else:
        buf = _nan_buffer(n, torch.float32 if flags & F_OUT_F32 else BF16, dev, guard=N)[0]
    buf2 = _nan_buffer(n, BF16, dev, guard=N)[0] if flags & (F_OUT2_RELU | F_OUT2_BF16) else None
    cos, sin, rope_cols, tpi, gw = rope if rope is not None else (None, None, 0, 0, 0)
    _call(lib.d3r_gemm_bf16(_p(ops['A']), _p(ops['W']), _p(buf), _p(ops['bias']), _p(ops['add0']), _p(buf2), M, N, K, N, flags,
                            _p(cos), _p(sin), rope_cols, tpi, gw, _lib.stream_ptr()))
    return buf, buf2


@pytest.mark.timeout(900)
@pytest.mark.parametrize('row', GEMM_TABLE, ids=[r[0] for r in GEMM_TABLE])
def test_gemm_matches_float64(cuda_device, gemm_family, row):
    """d3r_gemm_bf16 vs A B^T (+ epilogue) in float64 on the same bf16 operands, at the row's M cases.  Bound: _epilogue64's
    e; bf16 outputs by _check_bf16 (>= 99 % equal to bf16(ref)), fp32 outputs (F_OUT_F32, the residual stream) within e.
    The residual starts as residual_start (mixed signs, zeros of both signs, tiny and subnormal values).
    Resolution (each must be rejected): the last k16 slice of K dropped; A columns 3 and 11 swapped inside the first 64-wide
    k block; the bias rolled by one column; RoPE with the y and x positions swapped; v rotated too (rope_cols = N rows of a
    fused k|v projection); the fp32 residual rounded to bf16 before the add; GELU by the tanh approximation (fp32 output:
    at bf16 the output rounding hides it)."""
    dev = cuda_device
    lib = _lib.get_lib()
    name, N, K, flags, rope_cols, cases = row
    row_i = GEMM_TABLE.index(row)
    cos, sin = _rope_tables(dev)
    f32 = bool(flags & (F_OUT_F32 | F_RESID_INPLACE))
    for case_i, (B, gh, gw) in enumerate(cases):
        ops = _gemm_operands(row_i, case_i, N, K, flags, B, gh, gw, dev)
        M = ops['M']
        rope = (cos, sin, rope_cols, gh * gw, gw) if flags & F_ROPE else None
        buf, buf2 = _run_gemm(lib, ops, N, K, flags, rope, dev)
        out = buf[:M * N].view(M, N)
        A64, W64 = ops['A'].double(), ops['W'].double()
        P = A64 @ W64.T
        S = A64.abs() @ W64.abs().T
        b64 = ops['bias'].double() if ops['bias'] is not None else None
        a64 = ops['add0'].double() if ops['add0'] is not None else None
        r64 = ops['resid'].double() if ops['resid'] is not None else None
        kw = dict(bias=b64, add0=a64, rope=rope, resid=r64)
        ref, e = _epilogue64(P, S, K, flags, **kw)
        what = f'{name} impl={gemm_family} M={M} ({B}x{gh}x{gw}) N={N} K={K}'
        if f32:
            assert torch.isfinite(out).all(), f'{what}: non-finite or unwritten output'
            ratio, exact = _fp32_ratio(out, ref, e), float('nan')
            assert ratio <= 1.0, f'{what}: worst |err|/bound = {ratio:.3f}'
            bound = e + 1e-30
        else:
            ratio, exact, bound = _check_bf16(out, ref, e, what)
        assert _guard_ok(buf, M * N), f'{what}: the row after M was written'
        ratio2 = 0.0
        if buf2 is not None:
            out2 = buf2[:M * N].view(M, N)
            ratio2 = _check_bf16(out2, ref.clamp(min=0) if flags & F_OUT2_RELU else ref, e, f'{what} out2')[0]
            assert _guard_ok(buf2, M * N), f'{what}: out2 row after M was written'

        def epi(P_=P, **over):
            return _epilogue64(P_, S, K, flags, **dict(kw, **over))[0]

        checks = [('last k16 slice dropped', epi(P - A64[:, K - 16:] @ W64[:, K - 16:].T)),
                  ('A columns 3 and 11 swapped', epi(P + torch.outer(A64[:, 11] - A64[:, 3], W64[:, 3] - W64[:, 11])))]
        if b64 is not None:
            checks.append(('bias rolled by one column', epi(bias=b64.roll(1))))
        if rope is not None:
            checks.append(('RoPE y / x positions swapped', epi(swap_yx=True)))
            if 2 * rope_cols == N:
                checks.append(('v rotated too', epi(rope=(cos, sin, N, gh * gw, gw))))
        if r64 is not None:
            checks.append(('residual through bf16', epi(resid=ops['resid'].to(BF16).double())))
        if flags & F_GELU and f32:
            checks.append(('tanh GELU', epi(gelu='tanh')))
        for cname, bad in checks:
            assert _violations(out, bad, bound) > 0, f'{what}: {cname} not rejected'
        print(f'margin {what}: worst |err|/bound {ratio:.3f}' + (f', out2 {ratio2:.3f}' if buf2 is not None else '') +
              (f', exact {exact:.4f}' if not f32 else '') + f'; rejects: {", ".join(c for c, _ in checks)}')
        del P, S, ref, e, bound, checks


# ---- the implicit-GEMM 3x3 convolution (mode 1) ------------------------------------------------------------------------
def _conv_P(x64, w64, padding='zero'):
    """sum over the nine taps of x(b, y + ky - 1, x + kx - 1) w[:, :, ky, kx]^T = the unfold (im2col) product, one
    K = Cin slice per tap, -> (B H W, Cout).  padding='flat': the taps read the flattened pixel sequence, so that the left /
    right borders read the neighbouring row and the top / bottom rows the neighbouring image (zero only past the ends)."""
    B, H, W, Cin = x64.shape
    M = B * H * W
    P = torch.zeros((M, w64.shape[0]), dtype=F64, device=x64.device)
    if padding == 'zero':
        xp = F.pad(x64, (0, 0, 1, 1, 1, 1))
    else:
        xf = F.pad(x64.reshape(M, Cin), (0, 0, W + 1, W + 1))
    for ky in range(3):
        for kx in range(3):
            if padding == 'zero':
                xt = xp[:, ky:ky + H, kx:kx + W].reshape(M, Cin)
            else:
                o = (W + 1) + (ky - 1) * W + (kx - 1)
                xt = xf[o:o + M]
            P += xt @ w64[:, :, ky, kx].T
    return P


@pytest.mark.timeout(900)
@pytest.mark.parametrize('row', CONV_TABLE, ids=[r[0] for r in CONV_TABLE])
def test_conv3x3_matches_float64(cuda_device, gemm_family, row):
    """d3r_conv3x3_bf16 vs conv2d(padding=1) (+ epilogue) in float64 on the same bf16 operands, as the unfold product, at
    the row's (B, H, W) cases.  One K = 9 Cin reduction per output: e from _epilogue64 with g(9 Cin) and
    S = conv(|x|, |w|) + |bias|; out and out2 (= relu of the same value) by _check_bf16.
    Resolution: zero padding replaced by the flattened neighbour (left / right borders read the adjacent row, top / bottom
    rows the adjacent image); taps transposed (ky <-> kx); add1 dropped; for out2, the ReLU applied before the addends;
    image b > 0 reading image b - 1."""
    dev = cuda_device
    lib = _lib.get_lib()
    name, Cin, Cout, flags, cases = row
    row_i = CONV_TABLE.index(row)
    K = 9 * Cin
    for case_i, (B, H, W) in enumerate(cases):
        seed = 9000 + 100 * row_i + 10 * case_i
        x = _randn((B, H, W, Cin), seed, dev).to(BF16)
        w = _randn((Cout, Cin, 3, 3), seed + 1, dev, scale=K ** -0.5).to(BF16)
        wp = w.permute(0, 2, 3, 1).contiguous()                  # [Cout][ky][kx][Cin]
        bias = _randn((Cout,), seed + 2, dev).float() if flags & F_BIAS else None
        add0 = _randn((B, H, W, Cout), seed + 3, dev).to(BF16) if flags & F_ADD0 else None
        add1 = _randn((B, H, W, Cout), seed + 4, dev).to(BF16) if flags & F_ADD1 else None
        M = B * H * W
        n = M * Cout
        buf = _nan_buffer(n, BF16, dev, guard=W * Cout)[0]
        buf2 = _nan_buffer(n, BF16, dev, guard=W * Cout)[0] if flags & F_OUT2_RELU else None
        _call(lib.d3r_conv3x3_bf16(_p(x), _p(wp), _p(buf), _p(bias), _p(add0), _p(add1), _p(buf2), B, H, W, Cin, Cout, flags,
                                   _lib.stream_ptr()))
        x64, w64 = x.double(), w.double()
        P = _conv_P(x64, w64)
        S = _conv_P(x64.abs(), w64.abs())
        kw = dict(bias=bias.double() if bias is not None else None,
                  add0=add0.double().reshape(M, Cout) if add0 is not None else None,
                  add1=add1.double().reshape(M, Cout) if add1 is not None else None)
        ref, e = _epilogue64(P, S, K, flags, **kw)
        tw = 16
        while tw < W and tw < 128:
            tw *= 2
        what = f'{name} impl={gemm_family} B={B} {H}x{W} Cin={Cin} Cout={Cout} (tile {128 // tw}x{tw})'
        out = buf[:n].view(M, Cout)
        ratio, exact, bound = _check_bf16(out, ref, e, what)
        assert _guard_ok(buf, n), f'{what}: the pixel row after the last image was written'
        checks = [('flattened-neighbour padding', out, _epilogue64(_conv_P(x64, w64, 'flat'), S, K, flags, **kw)[0], bound),
                  ('taps transposed', out, _epilogue64(_conv_P(x64, w64.transpose(2, 3)), S, K, flags, **kw)[0], bound)]
        if add1 is not None:
            checks.append(('add1 dropped', out, _epilogue64(P, S, K, flags, **dict(kw, add1=None))[0], bound))
        ratio2 = 0.0
        if buf2 is not None:
            out2 = buf2[:n].view(M, Cout)
            ratio2, _, bound2 = _check_bf16(out2, ref.clamp(min=0), e, f'{what} out2')
            assert _guard_ok(buf2, n), f'{what}: out2 pixel row after the last image was written'
            if add0 is not None:
                early = _epilogue64(P, S, K, flags & ~(F_ADD0 | F_ADD1), **kw)[0].clamp(min=0) + kw['add0']
                if add1 is not None:
                    early = early + kw['add1']
                checks.append(('ReLU before the addends (out2)', out2, early, bound2))
        bad = ref.view(B, H * W, Cout).clone()
        bad[1:] = ref.view(B, H * W, Cout)[:-1]
        checks.append(('image b reading image b - 1', out, bad.view(M, Cout), bound))
        for cname, o, bad, bd in checks:
            assert _violations(o, bad, bd) > 0, f'{what}: {cname} not rejected'
        print(f'margin {what}: worst |err|/bound {ratio:.3f}' + (f', out2 {ratio2:.3f}' if buf2 is not None else '') +
              f', exact {exact:.4f}; rejects: {", ".join(c[0] for c in checks)}')
        del P, S, ref, e, bound, checks


# ---- bit identities: kernel families, store paths; instantiation coverage -----------------------------------------------
def _launch_key(rec, store):
    return (rec['tag'], int(re.search(r'epi=(\d+)', rec['detail']).group(1)), store if rec['tag'].endswith('_bn256') else None)


@pytest.mark.timeout(900)
def test_families_and_stores_bit_identical_and_cover_every_instantiation(cuda_device):
    """Every case of both tables: impl 0 (1-CTA kernels) and impl 1 (CTA pairs) run the same wgmma sequence on the same
    shared-memory layout, so they must give the same bits (guard rows included); for the GEMMs also the register-store
    (store 0) and TMA-store (store 1) epilogues, which the 256-wide specialised epilogues select between (bias-only bf16
    EPI_ACT of act_conv[3] / act3_down included).  The (profiler tag, epilogue, store) of every launch is recorded: the
    tables must reach every gemm_kernel instantiation that dispatch() in gemm_host.cu can launch (INSTANTIATIONS)."""
    dev = cuda_device
    lib = _lib.get_lib()
    cos, sin = _rope_tables(dev)
    seen, mismatches = set(), []

    def run(fn, store):
        lib.d3r_prof_enable(1)
        bufs = fn()
        recs = _lib.prof_dump()
        assert len(recs) == 1, recs
        seen.add(_launch_key(recs[0], store))
        return bufs

    try:
        for row_i, (name, N, K, flags, rope_cols, cases) in enumerate(GEMM_TABLE):
            for case_i, (B, gh, gw) in enumerate(cases):
                ops = _gemm_operands(row_i, case_i, N, K, flags, B, gh, gw, dev)
                rope = (cos, sin, rope_cols, gh * gw, gw) if flags & F_ROPE else None
                results = {}
                for impl in (0, 1):
                    for store in (0, 1):
                        lib.d3r_set_gemm_impl(impl)
                        lib.d3r_set_gemm_store(store)
                        results[impl, store] = run(lambda: _run_gemm(lib, ops, N, K, flags, rope, dev), store)
                base = results[0, 1]
                for key, bufs in results.items():
                    for a, b in zip(base, bufs):
                        if a is not None and not torch.equal(_bits(a), _bits(b)):
                            mismatches.append(f'{name} M={ops["M"]} impl/store {key} vs (0, 1): '
                                              f'{int((_bits(a) != _bits(b)).sum())} elements differ')
        lib.d3r_set_gemm_store(1)
        for row_i, (name, Cin, Cout, flags, cases) in enumerate(CONV_TABLE):
            for case_i, (B, H, W) in enumerate(cases):
                seed = 9000 + 100 * row_i + 10 * case_i
                x = _randn((B, H, W, Cin), seed, dev).to(BF16)
                wp = _randn((Cout, 3, 3, Cin), seed + 1, dev, scale=(9 * Cin) ** -0.5).to(BF16)
                bias = _randn((Cout,), seed + 2, dev).float() if flags & F_BIAS else None
                adds = [_randn((B, H, W, Cout), seed + s, dev).to(BF16) if flags & fl else None for s, fl in ((3, F_ADD0), (4, F_ADD1))]
                n = B * H * W * Cout

                def conv():
                    o = _nan_buffer(n, BF16, dev, guard=W * Cout)[0]
                    o2 = _nan_buffer(n, BF16, dev, guard=W * Cout)[0] if flags & F_OUT2_RELU else None
                    _call(lib.d3r_conv3x3_bf16(_p(x), _p(wp), _p(o), _p(bias), _p(adds[0]), _p(adds[1]), _p(o2), B, H, W, Cin, Cout,
                                               flags, _lib.stream_ptr()))
                    return o, o2

                results = []
                for impl in (0, 1):
                    lib.d3r_set_gemm_impl(impl)
                    results.append(run(conv, 1))
                for a, b in zip(*results):
                    if a is not None and not torch.equal(_bits(a), _bits(b)):
                        mismatches.append(f'{name} B={B} {H}x{W}: impl 1 vs 0: {int((_bits(a) != _bits(b)).sum())} elements differ')
    finally:
        lib.d3r_prof_enable(0)
        lib.d3r_set_gemm_impl(2)
        lib.d3r_set_gemm_store(1)
    assert not mismatches, '\n'.join(mismatches)
    missing = INSTANTIATIONS - seen
    assert not missing, f'instantiations no table row reaches: {sorted(missing, key=str)}'
    print(f'bit identities: {len(seen)} (tag, epilogue, store) combinations launched, all {len(INSTANTIATIONS)} instantiations')


# ---- the tables against the forward's own launches ---------------------------------------------------------------------
_DETAIL = re.compile(r'M=(\d+) N=(\d+) K=(\d+) flags=0x([0-9a-f]+) mode=(\d+) epi=(\d+)')


def _forward_launch_keys(records):
    """(N, K, flags, mode) of every gemm_kernel launch in a profiler dump, except the transposed conv and the head tail"""
    keys = set()
    for r in records:
        m = _DETAIL.fullmatch(r['detail'])
        if not (r['tag'].startswith(('gemm_', 'conv3x3_')) and m):
            continue
        N, K, fl, mode = int(m.group(2)), int(m.group(3)), int(m.group(4), 16), int(m.group(5))
        if not fl & (F_CONVT | F_HEAD_FINAL):
            keys.add((N, K, fl, mode))
    return keys


@pytest.mark.timeout(1200)
def test_tables_cover_the_forward_launches(cuda_device):
    """packed.forward on the published vitl_512_dpt at 512x384 and vitl_224_linear at 224 (B = 2 pairs, synthetic weights)
    with the profiler on: every (N, K, flags, mode) the forward launches gemm_kernel with (the transposed convs and the head
    tail aside) is a row of GEMM_TABLE / CONV_TABLE, and every forward row is launched by one of the two models.  A new GEMM
    call, or changed flags on one, fails here until the tables cover it."""
    import numpy as np
    from dust3r_b200.config import vitl_224_linear, vitl_512_dpt
    from dust3r_b200.utils.synth import synth_images
    from test_forward_gpu import _build
    dev = cuda_device
    keys = set()
    for cfg, H, W in ((vitl_512_dpt(), 384, 512), (vitl_224_linear(), 224, 224)):
        net, _ = _build(cfg, 0, dev)
        imgs = torch.cat([im['img'] for im in synth_images(4, H, W, seed=3)]).to(dev)
        packed = net.repack()
        _lib.prof_enable(True)
        try:
            packed.forward(imgs, np.arange(2, dtype=np.int32), 2 + np.arange(2, dtype=np.int32), 2, H, W)
            torch.cuda.synchronize()
            recs = _lib.prof_dump()
        finally:
            _lib.prof_enable(False)
        keys |= _forward_launch_keys(recs)
        del net, packed
    uncovered = keys - _table_keys()
    assert not uncovered, f'forward GEMM / conv launches (N, K, flags, mode) without a table row: {sorted(uncovered)}'
    forward_rows = ({(N, K, fl, 0) for _, N, K, fl, _, _ in GEMM_FORWARD} |
                    {(Cout, 9 * Cin, fl, 1) for _, Cin, Cout, fl, _ in CONV_FORWARD})
    unused = forward_rows - keys
    assert not unused, f'forward table rows the forward does not launch: {sorted(unused)}'
    print(f'forward launches: {len(keys)} distinct (N, K, flags, mode), all in the tables')


# ---- the forward under programmatic dependent launch ---------------------------------------------------------------------
_PDL_CHILD = r'''
import sys
import numpy as np
import torch
from dust3r_b200.config import vitl_512_dpt
from dust3r_b200.utils.synth import synth_images
from test_forward_gpu import _build
dev = torch.device('cuda:0')
net, _ = _build(vitl_512_dpt(), 0, dev)
imgs = torch.cat([im['img'] for im in synth_images(4, 384, 512, seed=3)]).to(dev)
r1, r2 = net.repack().forward(imgs, np.arange(2, dtype=np.int32), 2 + np.arange(2, dtype=np.int32), 2, 384, 512)
torch.cuda.synchronize()
torch.save({k: v.cpu() for k, v in (('pts1', r1['pts3d']), ('conf1', r1['conf']), ('pts2', r2['pts3d']), ('conf2', r2['conf']))},
           sys.argv[1])
'''


@pytest.mark.timeout(1200)
def test_forward_with_pdl_is_bit_identical(cuda_device, tmp_path):
    """D3R_PDL=1 launches every forward kernel with programmatic dependent launch; each kernel waits for its predecessor
    before it touches memory another kernel writes, so pts3d and conf must equal the D3R_PDL=0 run's bits (vitl_512_dpt,
    B = 2, 512x384, same device).  pdl::enabled() reads the environment once per process, so each setting runs in a child
    process, once, under a timeout that kills it."""
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(tests_dir)
    torch.cuda.empty_cache()
    res = {}
    for pdl in ('0', '1'):
        env = dict(os.environ, D3R_PDL=pdl, PYTHONPATH=os.pathsep.join([root, tests_dir] + ([os.environ['PYTHONPATH']] if
                                                                                         os.environ.get('PYTHONPATH') else [])))
        out = tmp_path / f'pdl{pdl}.pt'
        cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', _PDL_CHILD, str(out)]
        p = subprocess.run(cmd, env=env, cwd=root, capture_output=True, text=True, timeout=900)
        assert p.returncode == 0, f'D3R_PDL={pdl} child failed ({p.returncode}):\n{p.stderr[-4000:]}'
        res[pdl] = torch.load(out)
    for k in ('pts1', 'conf1', 'pts2', 'conf2'):
        a, b = res['0'][k], res['1'][k]
        assert torch.isfinite(a).all(), k
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f'{k}: {int((a != b).sum())} elements differ with PDL'
    print('forward with D3R_PDL=1 == D3R_PDL=0 bit for bit (pts3d, conf of both views)')
