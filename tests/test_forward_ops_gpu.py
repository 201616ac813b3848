"""The forward's glue kernels, its transposed convolution and its fused DPT head tail, one at a time, against float64 torch on
the same inputs; attention against float64 with a bound that can see a one-key error, and its two implementations bit for bit.

Every bound is per element, derived from the rounding of the kernel's own arithmetic (worked out in each test's docstring),
and scales with the element's own magnitude or its sum's sum of |terms|.  Notation:
  U = 2^-8      unit roundoff of bf16 (8 significant bits, round to nearest even): |bf16(y) - y| <= U |y|;
  g(K)          fp32 accumulation of a K-long wgmma reduction: (K/16 + 8) * 2^-23 * sum|terms| -- one fp32 rounding per k16
                step into the accumulator, plus a few for the products of one step, the bias and the epilogue, doubled;
  bf16 outputs: |out - ref64| <= U (|ref64| + e) + e, e = the fp32 error before the final rounding.
Each test also computes a reference perturbed by a named small bug and asserts that its bound rejects it, and prints its worst
|err| / bound (pytest -s or -rP).  Outputs start as NaN so that an unwritten element fails; guard elements after every output
must keep their value."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from dust3r_b200 import _lib

U = 2.0 ** -8
F64 = torch.float64
# token grids of the published inputs: 512x384, 512x336, 512x288, 512x256, 512x160, 224x224, and the portrait 336x512, 384x512
GRIDS = [(24, 32), (21, 32), (18, 32), (16, 32), (10, 32), (14, 14), (32, 21), (32, 24)]
GUARD = -7.0


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _call(rc):
    _lib.check(rc)
    torch.cuda.synchronize()


def _randn(shape, seed, dev, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=F64) * scale).to(dev)


def _gamma(K):
    return (K / 16 + 8) * 2.0 ** -23


def _nan_buffer(n, dtype, dev, guard=64):
    """flat buffer of n NaNs followed by `guard` guard elements; returns (buffer, view of the first n)"""
    buf = torch.full((n + guard,), float('nan'), dtype=dtype, device=dev)
    buf[n:] = GUARD
    return buf, buf[:n]


def _guard_ok(buf, n):
    return bool((buf[n:].double() == GUARD).all())


def _bf16_bound(ref, e):
    return U * (ref.abs() + e) + e + 1e-30


def _violations(out, ref, bound):
    return int(((out.double() - ref).abs() > bound).sum())


def _check_bf16(out, ref, e, what, min_exact=0.99, exact_mask=None):
    """|out - ref| <= U (|ref| + e) + e everywhere; at least `min_exact` of the elements (under exact_mask) equal bf16(ref)."""
    assert torch.isfinite(out.double()).all(), f'{what}: non-finite or unwritten output'
    bound = _bf16_bound(ref, e)
    ratio = ((out.double() - ref).abs() / bound).max().item()
    assert ratio <= 1.0, f'{what}: worst |err|/bound = {ratio:.3f}'
    eq = out == ref.to(torch.bfloat16)
    if exact_mask is not None:
        eq = eq[exact_mask]
    exact = eq.double().mean().item() if eq.numel() else 1.0
    assert exact >= min_exact, f'{what}: only {exact:.4f} of the elements equal bf16(ref)'
    return ratio, exact, bound


@pytest.fixture(params=[0, 1], ids=['cta1', 'cta_pair'])
def gemm_family(request):
    """1-CTA kernels / CTA-pair kernels (restored to the default policy afterwards)"""
    lib = _lib.get_lib()
    lib.d3r_set_gemm_impl(request.param)
    try:
        yield request.param
    finally:
        lib.d3r_set_gemm_impl(2)


# ---- LayerNorm ---------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(300)
@pytest.mark.parametrize('M,C', [(777, 1024), (1537, 768), (3, 768), (9, 2048)])
def test_layernorm_matches_float64(cuda_device, M, C):
    """d3r_layernorm_bf16 vs F.layer_norm in float64 on the same fp32 rows.

    Kernel: one warp per row, each lane sums C/32 values, then a 5-level shuffle tree, mean = s / C; the variance is the same
    sum over (x - mean)^2; rstd = rsqrtf(var + eps) (<= 2 ulp); y = (x - mean) * rstd * g + b, rounded to bf16.  So
      |mean - mu| <= dmu = (C/32 + 7) 2^-24 mean|x|,   rel. error of rstd <= er = (C/32 + 12) 2^-25 + 2^-22 + dmu^2 / (var + eps),
      e = rstd |g| (|x - mu| er + dmu) + 2^-22 (|xhat g| + |b|).
    Rows: plain N(0, 1); a common offset of 300 or -1000 (mean >> std: cancellation); std 1e-3 ~ sqrt(eps) around 0.5 (where
    eps matters); constant rows (variance 0, exact mean: y = b).  At least 99 % of the plain rows' elements equal bf16(ref).
    Resolution: eps added outside the square root, rstd = 1 / (sqrt(var) + eps), is rejected."""
    dev = cuda_device
    lib = _lib.get_lib()
    eps = 1e-6
    x = _randn((M, C), 1, dev)
    cls = torch.arange(M, device=dev) % 8
    x[cls == 0] = 300.0 + x[cls == 0]
    x[cls == 1] = 0.5 + 1e-3 * x[cls == 1]
    x[cls == 2] = 3.5
    x[cls == 3] = -1000.0 + 2.0 * x[cls == 3]
    x[cls == 4] = -0.75
    x32 = x.float().contiguous()
    x64 = x32.double()
    g32 = (1.0 + 0.2 * _randn((C,), 2, dev)).float()
    b32 = (0.3 * _randn((C,), 3, dev)).float()
    g64, b64 = g32.double(), b32.double()
    buf, out = _nan_buffer(M * C, torch.bfloat16, dev, guard=3 * C)
    _call(lib.d3r_layernorm_bf16(_p(x32), _p(g32), _p(b32), _p(out), M, C, eps, _lib.stream_ptr()))
    out = out.view(M, C)
    ref = F.layer_norm(x64, (C,), g64, b64, eps)
    mu = x64.mean(1, keepdim=True)
    xc = x64 - mu
    var = (xc * xc).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    dmu = (C / 32 + 7) * 2.0 ** -24 * x64.abs().mean(1, keepdim=True)
    er = (C / 32 + 12) * 2.0 ** -25 + 2.0 ** -22 + dmu * dmu / (var + eps)
    e = rstd * g64.abs() * (xc.abs() * er + dmu) + 2.0 ** -22 * ((xc * rstd * g64).abs() + b64.abs())
    ratio, exact, bound = _check_bf16(out, ref, e, f'layernorm M={M} C={C}', exact_mask=(cls >= 5)[:, None].expand(M, C))
    assert _guard_ok(buf, M * C)
    assert torch.equal(out[cls == 2], b32.to(torch.bfloat16).expand_as(out[cls == 2]))   # constant rows: y = b exactly
    bad = xc / (torch.sqrt(var) + eps) * g64 + b64
    assert _violations(out, bad, bound) > 0, 'eps outside the square root not rejected'
    print(f'margin layernorm M={M} C={C}: worst |err|/bound {ratio:.3f}, exact {exact:.4f}')


# ---- bilinear x2 upsample ----------------------------------------------------------------------------------------------
def _upsample_ref(x64, Ho, Wo, full=None):
    """x64 (B,H,W,C).  The top-left Ho x Wo of the align_corners=True bilinear resize to `full` (default (2H, 2W)), the sum of
    |terms| S = sum w |corner| and L = the largest |x| in the 3x3 input neighbourhood of the output's top-left corner."""
    B, H, W, Cc = x64.shape
    Hf, Wf = full if full is not None else (2 * H, 2 * W)

    def coords(n_out, n_in, n_full):
        s = torch.arange(n_out, dtype=F64, device=x64.device) * ((n_in - 1) / (n_full - 1) if n_full > 1 else 0.0)
        i0 = s.floor().long().clamp(max=n_in - 1)
        return i0, (i0 + 1).clamp(max=n_in - 1), s - i0

    y0, y1, fy = coords(Ho, H, Hf)
    x0, x1, fx = coords(Wo, W, Wf)
    fy, fx = fy.view(1, Ho, 1, 1), fx.view(1, 1, Wo, 1)
    ra, rb = x64[:, y0], x64[:, y1]
    c00, c01, c10, c11 = ra[:, :, x0], ra[:, :, x1], rb[:, :, x0], rb[:, :, x1]
    w00, w01, w10, w11 = (1 - fy) * (1 - fx), (1 - fy) * fx, fy * (1 - fx), fy * fx
    ref = w00 * c00 + w01 * c01 + w10 * c10 + w11 * c11
    S = w00 * c00.abs() + w01 * c01.abs() + w10 * c10.abs() + w11 * c11.abs()
    mp = F.max_pool2d(x64.abs().permute(0, 3, 1, 2), 3, 1, 1).permute(0, 2, 3, 1)
    L = mp[:, y0][:, :, x0]
    return ref, S, L


def _upsample_cases():
    cases = []
    for gh, gw in GRIDS:
        h3, w3 = (gh + 1) // 2, (gw + 1) // 2
        cases.append((3, h3, w3, 256, gh, gw))                  # refinenet4: cropped to the level-2 size when gh / gw is odd
        cases.append((3, gh, gw, 256, 2 * gh, 2 * gw))
        cases.append((3, 2 * gh, 2 * gw, 256, 4 * gh, 4 * gw))
        cases.append((3, 4 * gh, 4 * gw, 256, 8 * gh, 8 * gw))
        cases.append((3, 8 * gh, 8 * gw, 128, 16 * gh, 16 * gw))  # the head's upsample
    return cases


@pytest.mark.timeout(900)
@pytest.mark.parametrize('grid', GRIDS + ['edges'], ids=[f'{a}x{b}' for a, b in GRIDS] + ['edges'])
def test_upsample2x_matches_float64(cuda_device, grid):
    """d3r_upsample2x_bf16 vs F.interpolate(x2, bilinear, align_corners=True)[..., :Ho, :Wo] in float64, at every level of
    run_dpt for the grid (B = 3), or at the degenerate edges H = 1 / W = 1.

    Kernel: source coordinate sx = ox * fl((W-1) / (2W-1)) in fp32, so |dsx| <= 2^-23 W (same on y); weights
    (1-fy)(1-fx), ... and the 4-term sum in fp32.  A coordinate error moves the output by at most 2 L per unit (L = largest
    |x| of the neighbourhood, which also covers a truncation to the previous cell), so
      e = 2^-21 S + 2^-22 (H + W) L,   S = sum of w |corner|.
    Resolution: the last output row taking the previous row's weights; the crop taken from a resize to (Ho, Wo) instead of
    (2H, 2W); image b > 0 reading image b - 1."""
    dev = cuda_device
    lib = _lib.get_lib()
    cases = _upsample_cases() if grid != 'edges' else [(3, 1, 7, 128, 2, 14), (3, 5, 1, 64, 9, 2), (4, 1, 1, 256, 2, 1),
                                                          (3, 2, 3, 8, 3, 5), (3, 3, 3, 128, 6, 5)]
    for i, (B, H, W, Cc, Ho, Wo) in enumerate(cases):
        x = _randn((B, H, W, Cc), 10 + i, dev).to(torch.bfloat16)
        x64 = x.double()
        n = B * Ho * Wo * Cc
        buf, out = _nan_buffer(n, torch.bfloat16, dev, guard=Wo * Cc)
        _call(lib.d3r_upsample2x_bf16(_p(x), _p(out), B, H, W, Cc, Ho, Wo, _lib.stream_ptr()))
        out = out.view(B, Ho, Wo, Cc)
        ref, S, L = _upsample_ref(x64, Ho, Wo)
        tv = F.interpolate(x64.permute(0, 3, 1, 2), size=(2 * H, 2 * W), mode='bilinear', align_corners=True)
        assert (tv[:, :, :Ho, :Wo].permute(0, 2, 3, 1) - ref).abs().max().item() < 1e-12   # the explicit reference is F.interpolate
        e = 2.0 ** -21 * S + 2.0 ** -22 * (H + W) * L
        what = f'upsample B={B} {H}x{W}x{Cc} -> {Ho}x{Wo}'
        ratio, exact, bound = _check_bf16(out, ref, e, what)
        assert _guard_ok(buf, n), what
        if H > 1 and Ho > 1:
            bad = ref.clone()
            bad[:, Ho - 1] = ref[:, Ho - 2]
            assert _violations(out, bad, bound) > 0, f'{what}: last row with the previous row\'s weights not rejected'
        if (Ho, Wo) != (2 * H, 2 * W) and Ho > 1 and Wo > 1:
            bad = _upsample_ref(x64, Ho, Wo, full=(Ho, Wo))[0]
            assert _violations(out, bad, bound) > 0, f'{what}: crop of a ({Ho}, {Wo}) resize not rejected'
        bad = ref.clone()
        bad[1:] = ref[:-1]
        assert _violations(out, bad, bound) > 0, f'{what}: batch shift not rejected'
        print(f'margin {what}: worst |err|/bound {ratio:.3f}, exact {exact:.4f}')


# ---- pure data movement: strided 3x3 im2col, patch im2col ----------------------------------------------------------------
@pytest.mark.timeout(300)
def test_im2col_3x3_s2_bitwise(cuda_device):
    """d3r_im2col_3x3_s2_bf16 == F.unfold(k=3, s=2, p=1) reordered to the forward's [pixel][tap][C], bit for bit, at the
    act_postprocess[3] shape of every grid (C = 768, B = 3) and at 1-pixel edges.  Resolution: taps in (kx, ky) order."""
    dev = cuda_device
    lib = _lib.get_lib()
    cases = [(3, gh, gw, 768) for gh, gw in GRIDS] + [(3, 1, 1, 8), (3, 1, 5, 16), (2, 7, 1, 8), (3, 2, 2, 64)]
    for i, (B, H, W, Cc) in enumerate(cases):
        x = _randn((B, H, W, Cc), 40 + i, dev).to(torch.bfloat16)
        Ho, Wo = (H + 1) // 2, (W + 1) // 2
        n = B * Ho * Wo * 9 * Cc
        buf, out = _nan_buffer(n, torch.bfloat16, dev, guard=9 * Cc)
        _call(lib.d3r_im2col_3x3_s2_bf16(_p(x), _p(out), B, H, W, Cc, _lib.stream_ptr()))
        cols = F.unfold(x.float().permute(0, 3, 1, 2), 3, padding=1, stride=2).view(B, Cc, 3, 3, Ho * Wo)
        ref = cols.permute(0, 4, 2, 3, 1).reshape(-1).to(torch.bfloat16)
        what = f'im2col_s2 B={B} {H}x{W}x{Cc}'
        assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), what
        assert _guard_ok(buf, n), what
        if H == 1 and W == 1:
            continue                                      # only the centre tap is inside the image: symmetric
        bad = cols.permute(0, 4, 3, 2, 1).reshape(-1).to(torch.bfloat16)
        assert not torch.equal(out.view(torch.int16), bad.view(torch.int16)), f'{what}: transposed taps not rejected'


@pytest.mark.timeout(300)
def test_patch_im2col16_bitwise(cuda_device):
    """d3r_patch_im2col16 == F.unfold(k=16, s=16) -> bf16 (round to nearest even), bit for bit, for the images of every grid
    (B = 3).  Some pixels sit exactly halfway between two bf16 values (ties go to even).  Resolution: px / py swapped."""
    dev = cuda_device
    lib = _lib.get_lib()
    for i, (gh, gw) in enumerate(GRIDS):
        B, H, W = 3, 16 * gh, 16 * gw
        img = _randn((B, 3, H, W), 60 + i, dev).float()
        lo = img.to(torch.bfloat16)
        hi = (lo.view(torch.int16) + 1).view(torch.bfloat16)
        tie = ((lo.float() + hi.float()) / 2).contiguous()               # exactly halfway, representable in fp32
        sel = (torch.arange(img.numel(), device=dev) % 7 == 0).view_as(img)
        img = torch.where(sel, tie, img).contiguous()
        n = B * gh * gw * 768
        buf, out = _nan_buffer(n, torch.bfloat16, dev, guard=768)
        _call(lib.d3r_patch_im2col16(_p(img), _p(out), B, H, W, _lib.stream_ptr()))
        cols = F.unfold(img, 16, stride=16).transpose(1, 2)             # (B, L, 3*16*16), c*256 + py*16 + px
        ref = cols.reshape(-1).to(torch.bfloat16)
        what = f'patch_im2col B={B} {H}x{W}'
        assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), what
        assert _guard_ok(buf, n), what
        bad = cols.reshape(B, gh * gw, 3, 16, 16).transpose(-1, -2).reshape(-1).to(torch.bfloat16)
        assert not torch.equal(out.view(torch.int16), bad.view(torch.int16)), f'{what}: px / py swap not rejected'


# ---- pointmap postprocess (shared by the linear head and the DPT head tail) -----------------------------------------------
CONF_MODES = [(0, 0.0, 0.0), (1, 1.0, 3.0e38), (1, 1.0, 20.0), (2, 0.5, 2.5)]


def _postprocess64(z, depth_mode, conf_mode, cmin, cmax):
    """dust3r/heads/postprocess.py in float64: z (..., 4) -> pts (..., 3), conf (...)"""
    xyz = z[..., :3]
    if depth_mode == 0:
        pts = xyz
    else:
        d = xyz.norm(dim=-1, keepdim=True)
        pts = xyz / d.clamp(min=1e-8) * (d * d if depth_mode == 1 else torch.expm1(d))
    c = z[..., 3]
    if conf_mode == 1:
        conf = cmin + c.exp().clamp(max=cmax - cmin)
    elif conf_mode == 2:
        conf = (cmax - cmin) * torch.sigmoid(c) + cmin
    else:
        conf = None
    return pts, conf


def _pts_bound(ref_pts, z, ez, depth_mode):
    """per pixel: L(d) * E + 2^-20 (1 + d) |ref|, E = sum of the xyz input errors, L the Lipschitz constant of the depth map
    (1 linear, 2 (d + E) square, exp(d + E) exp); 2^-20 (1 + d) covers ~8 fp32 roundings, sqrtf and expm1f (1 ulp) with its
    condition number d e^d / expm1(d) <= 1 + d."""
    d = z[..., :3].norm(dim=-1)
    E = ez[..., :3].sum(-1) if ez is not None else torch.zeros_like(d)
    Lc = torch.ones_like(d) if depth_mode == 0 else (2 * (d + E) if depth_mode == 1 else torch.exp(d + E))
    return Lc * E + 2.0 ** -20 * (1 + d) * ref_pts.norm(dim=-1) + 1e-30


def _conf_bound(ref_conf, z, ez, conf_mode, cmin, cmax):
    """exp: e^(c + e) e (unclipped slope), sigmoid: (cmax - cmin) / 4 * e; plus 2^-20 (|ref| + |cmin|) for expf / the sums"""
    e = ez[..., 3] if ez is not None else torch.zeros_like(z[..., 3])
    slope = torch.exp(z[..., 3] + e) if conf_mode == 1 else torch.full_like(e, (cmax - cmin) / 4)
    return slope * e + 2.0 ** -20 * (ref_conf.abs() + abs(cmin)) + 1e-30


def _check_pts_conf(pts, conf, ref_pts, ref_conf, pb, cb, what):
    assert torch.isfinite(pts).all(), f'{what}: non-finite or unwritten pts3d'
    rp = ((pts.double() - ref_pts).abs().amax(-1) / pb).max().item()
    assert rp <= 1.0, f'{what}: pts3d worst |err|/bound = {rp:.3f}'
    rc = 0.0
    if ref_conf is not None:
        assert torch.isfinite(conf).all(), f'{what}: non-finite or unwritten conf'
        rc = ((conf.double() - ref_conf).abs() / cb).max().item()
        assert rc <= 1.0, f'{what}: conf worst |err|/bound = {rc:.3f}'
    return rp, rc


def _pts_violations(pts, bad_pts, pb):
    return int(((pts.double() - bad_pts).abs().amax(-1) > pb).sum())


@pytest.mark.timeout(600)
@pytest.mark.parametrize('depth_mode', [0, 1, 2], ids=['linear', 'square', 'exp'])
@pytest.mark.parametrize('nch,conf_mode,cmin,cmax', [(3, 1, 1.0, 3.0e38), (4, 0, 0.0, 0.0)] + [(4,) + c for c in CONF_MODES[1:]])
def test_linear_head_postprocess_matches_float64(cuda_device, depth_mode, nch, conf_mode, cmin, cmax):
    """d3r_linear_head_postprocess vs pixel_shuffle + heads/postprocess.py in float64 on the same fp32 features, every grid,
    B = 3.  Per pixel: the linear depth mode copies (bit for bit), the others are within the relative bound of _pts_bound;
    conf within _conf_bound.  Pixels with zero xyz (the max(d, 1e-8) path) and with |xyz| ~ 1e-9 are included.  Without a
    confidence channel or with conf_mode 0, the conf buffer is not written.  Resolution: px and py swapped in the pixel
    shuffle; image b > 0 reading image b - 1."""
    dev = cuda_device
    lib = _lib.get_lib()
    writes_conf = nch == 4 and conf_mode != 0
    for i, (gh, gw) in enumerate(GRIDS):
        B, H, W = 3, 16 * gh, 16 * gw
        feat = _randn((B * gh * gw, nch, 256), 80 + i, dev)
        feat[::5, :3, 17] = 0.0                         # zero-norm pixels
        feat[1::7, :3, 200] *= 1e-9                     # tiny norms
        feat = feat.reshape(B * gh * gw, nch * 256).float().contiguous()
        pbuf, pts = _nan_buffer(B * H * W * 3, torch.float32, dev)
        cbuf, conf = _nan_buffer(B * H * W, torch.float32, dev)
        _call(lib.d3r_linear_head_postprocess(_p(feat), _p(pts), _p(conf), B, gh, gw, nch, depth_mode, conf_mode, cmin, cmax,
                                              _lib.stream_ptr()))
        pts, conf = pts.view(B, H, W, 3), conf.view(B, H, W)
        f64 = feat.double().view(B, gh, gw, nch * 256).permute(0, 3, 1, 2)
        z = F.pixel_shuffle(f64, 16).permute(0, 2, 3, 1)            # (B, H, W, nch)
        if nch == 3:
            z = torch.cat((z, torch.zeros_like(z[..., :1])), -1)
        ref_pts, ref_conf = _postprocess64(z, depth_mode, conf_mode if writes_conf else 0, cmin, cmax)
        what = f'linear head {gh}x{gw} nch={nch} depth={depth_mode} conf={conf_mode}'
        pb = _pts_bound(ref_pts, z, None, depth_mode)
        cb = _conf_bound(ref_conf, z, None, conf_mode, cmin, cmax) if writes_conf else None
        rp, rc = _check_pts_conf(pts, conf, ref_pts, ref_conf, pb, cb, what)
        if depth_mode == 0:
            assert torch.equal(pts, z[..., :3].float()), what
        assert int((ref_pts.norm(dim=-1) == 0).sum()) >= B * 16, f'{what}: no zero-norm pixels'
        assert _guard_ok(pbuf, B * H * W * 3), what
        if writes_conf:
            assert _guard_ok(cbuf, B * H * W), what
        else:
            assert torch.isnan(conf).all() and _guard_ok(cbuf, B * H * W), f'{what}: conf written without a confidence output'
        zt = F.pixel_shuffle(f64.reshape(B, nch, 16, 16, gh, gw).transpose(2, 3).reshape(B, nch * 256, gh, gw), 16)
        zt = zt.permute(0, 2, 3, 1)
        bad_pts = _postprocess64(torch.cat((zt, torch.zeros_like(zt[..., :1])), -1) if nch == 3 else zt, depth_mode, 0, 0, 0)[0]
        assert _pts_violations(pts, bad_pts, pb) > 0, f'{what}: px / py swap not rejected'
        bad_pts = ref_pts.clone()
        bad_pts[1:] = ref_pts[:-1]
        assert _pts_violations(pts, bad_pts, pb) > 0, f'{what}: batch shift not rejected'
        print(f'margin {what}: pts worst |err|/bound {rp:.3f}, conf {rc:.3f}')


# ---- transposed convolution (F_CONVT) ------------------------------------------------------------------------------------
@pytest.mark.timeout(600)
@pytest.mark.parametrize('Cin,k', [(96, 4), (192, 2)])
def test_conv_transpose_matches_float64(cuda_device, gemm_family, Cin, k):
    """d3r_conv_transpose_bf16 vs F.conv_transpose2d(stride=k) in float64 on the same bf16 operands: act_postprocess[0] / [1]
    of run_dpt (Cout = Cin) at every grid, B = 3, and 1-pixel edges.  Weights are generated in torch's (Cin, Cout, k, k) layout
    and packed with the permute the model uses.  Each output is one K = Cin dot product + bias: e = g(Cin) S,
    S = conv_transpose2d(|x|, |w|) + |bias|.  At least 99 % of the elements equal bf16(ref).
    Resolution: the bias indexed one channel off; image b > 0 reading image b - 1."""
    dev = cuda_device
    lib = _lib.get_lib()
    Cout = Cin
    cases = [(3, gh, gw) for gh, gw in GRIDS] + [(4, 1, 1), (3, 1, 7), (3, 5, 1)]
    for i, (B, h, w) in enumerate(cases):
        x = _randn((B, h, w, Cin), 100 + i, dev).to(torch.bfloat16)
        wt = _randn((Cin, Cout, k, k), 200 + i, dev, scale=Cin ** -0.5).to(torch.bfloat16)
        bias = _randn((Cout,), 300 + i, dev).float()
        wp = wt.permute(2, 3, 1, 0).reshape(k * k * Cout, Cin).contiguous()
        n = B * h * k * w * k * Cout
        buf, out = _nan_buffer(n, torch.bfloat16, dev, guard=k * Cout)
        _call(lib.d3r_conv_transpose_bf16(_p(x), _p(wp), _p(out), _p(bias), B, h, w, Cin, Cout, k, _lib.stream_ptr()))
        out = out.view(B, h * k, w * k, Cout)
        x64 = x.double().permute(0, 3, 1, 2)
        ref = F.conv_transpose2d(x64, wt.double(), bias.double(), stride=k).permute(0, 2, 3, 1)
        S = F.conv_transpose2d(x64.abs(), wt.double().abs(), bias.double().abs(), stride=k).permute(0, 2, 3, 1)
        what = f'conv_transpose impl={gemm_family} B={B} {h}x{w}x{Cin} k={k}'
        ratio, exact, bound = _check_bf16(out, ref, _gamma(Cin) * S, what)
        assert _guard_ok(buf, n), what
        b64 = bias.double()
        bad = ref + (b64.roll(-1) - b64)
        assert _violations(out, bad, bound) > 0, f'{what}: bias one channel off not rejected'
        bad = ref.clone()
        bad[1:] = ref[:-1]
        assert _violations(out, bad, bound) > 0, f'{what}: batch shift not rejected'
        print(f'margin {what}: worst |err|/bound {ratio:.3f}, exact {exact:.4f}')


# ---- DPT head tail (F_HEAD_FINAL) ----------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
@pytest.mark.parametrize('grid', GRIDS + [(0, 0)], ids=[f'{a}x{b}' for a, b in GRIDS] + ['5x7px'])
def test_conv3x3_head_tail_matches_float64(cuda_device, gemm_family, grid):
    """d3r_conv3x3_head_tail vs conv2d 128->128 (+ bias) -> ReLU -> 1x1 to 4 channels -> postprocess.py, all in float64 on the
    same bf16 / fp32 inputs, at the head resolution 16 gh x 16 gw of every grid (up to 512 x 384; widths 336 and 224 give
    ragged conv tiles), B = 3, plus a 5 x 7 pixel map; every depth mode x conf mode; a random head bias and one that is zero
    on xyz, with a zero input block and a negative conv bias, so that those pixels have xyz = 0 exactly (max(d, 1e-8)).

    Bound: conv channel c: e_c = g(1152) S_c, S_c = conv2d(|x|, |w|) + |bias|; ReLU is 1-Lipschitz; the 1x1 conv sums 128
    products per output in fp32 (32 per thread + 2 shuffles): e_z = sum_c |w4| e_c + 2^-18 (sum_c |w4| relu(y_c) + |b4|);
    then _pts_bound / _conf_bound per pixel.  Resolution: the 1x1 conv applied before the ReLU; image b > 0 reading b - 1."""
    dev = cuda_device
    lib = _lib.get_lib()
    gh, gw = grid
    B, H, W = (3, 16 * gh, 16 * gw) if gh else (3, 5, 7)
    seed = 500 + gh * 40 + gw
    x = _randn((B, H, W, 128), seed, dev)
    x[:, 8:14, 8:14] = 0.0
    x[:, -4:, -4:] = 0.0                                   # a zero block on the bottom-right border
    x = x.to(torch.bfloat16)
    wt = _randn((128, 128, 3, 3), seed + 1, dev, scale=1152 ** -0.5).to(torch.bfloat16)
    bias = (-0.05 - 0.3 * _randn((128,), seed + 2, dev).abs()).float()
    w4 = _randn((4, 128), seed + 3, dev, scale=128 ** -0.5).float().contiguous()
    wp = wt.permute(0, 2, 3, 1).contiguous()              # [Cout][ky][kx][Cin]
    x64 = x.double().permute(0, 3, 1, 2)
    y = F.conv2d(x64, wt.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    S = F.conv2d(x64.abs(), wt.double().abs(), bias.double().abs(), padding=1).permute(0, 2, 3, 1)
    r = y.clamp(min=0)
    aw4 = w4.double().abs()
    ec = _gamma(9 * 128) * S
    del S
    worst = [0.0, 0.0]
    for b4_kind in ('random', 'zero_xyz'):
        b4 = _randn((4,), seed + 4, dev).float()
        if b4_kind == 'zero_xyz':
            b4[:3] = 0.0
        z = r @ w4.double().T + b4.double()
        ez = ec @ aw4.T + 2.0 ** -18 * (r @ aw4.T + b4.double().abs())
        zbad = (y @ w4.double().T + b4.double()).clamp(min=0)
        for depth_mode in (0, 1, 2):
            for conf_mode, cmin, cmax in CONF_MODES:
                pbuf, pts = _nan_buffer(B * H * W * 3, torch.float32, dev)
                cbuf, conf = _nan_buffer(B * H * W, torch.float32, dev)
                _call(lib.d3r_conv3x3_head_tail(_p(x), _p(wp), _p(bias), _p(w4), _p(b4), _p(pts), _p(conf), B, H, W, depth_mode,
                                                conf_mode, cmin, cmax, _lib.stream_ptr()))
                pts, conf = pts.view(B, H, W, 3), conf.view(B, H, W)
                ref_pts, ref_conf = _postprocess64(z, depth_mode, conf_mode, cmin, cmax)
                what = f'head tail impl={gemm_family} B={B} {H}x{W} b4={b4_kind} depth={depth_mode} conf={conf_mode}'
                pb = _pts_bound(ref_pts, z, ez, depth_mode)
                cb = _conf_bound(ref_conf, z, ez, conf_mode, cmin, cmax) if conf_mode else None
                rp, rc = _check_pts_conf(pts, conf, ref_pts, ref_conf, pb, cb, what)
                worst = [max(worst[0], rp), max(worst[1], rc)]
                assert _guard_ok(pbuf, B * H * W * 3), what
                if conf_mode:
                    assert _guard_ok(cbuf, B * H * W), what
                else:
                    assert torch.isnan(conf).all() and _guard_ok(cbuf, B * H * W), f'{what}: conf written with conf_mode 0'
                if b4_kind == 'zero_xyz':
                    zn = ref_pts.norm(dim=-1) == 0
                    assert int(zn.sum()) >= 4 * B, f'{what}: no zero-norm pixels'
                    assert bool((pts[zn] == 0).all()), f'{what}: zero-norm pixels'
                bad_pts = _postprocess64(zbad, depth_mode, 0, 0, 0)[0]
                assert _pts_violations(pts, bad_pts, pb) > 0, f'{what}: 1x1 conv before the ReLU not rejected'
                bad_pts = ref_pts.clone()
                bad_pts[1:] = ref_pts[:-1]
                assert _pts_violations(pts, bad_pts, pb) > 0, f'{what}: batch shift not rejected'
    print(f'margin head tail impl={gemm_family} B={B} {H}x{W}: pts worst |err|/bound {worst[0]:.3f}, conf {worst[1]:.3f}')


# ---- attention -----------------------------------------------------------------------------------------------------------
ATTN_CASES = [
    # B, heads, Nq, Nk, layout
    (2, 16, 768, 768, 'self'),      # encoder: packed qkv, ld = 3 * 1024, 24 x 32 grid
    (3, 12, 672, 672, 'self'),      # decoder: packed qkv, ld = 3 * 768, 21 x 32 grid
    (2, 12, 768, 672, 'cross'),     # 512x384 queries against 512x336 keys: q ld = 768, k / v ld = 2 * 768
    (2, 12, 672, 768, 'cross'),
    (24, 12, 196, 196, 'self'),     # 576 tiles: several rounds per persistent CTA
    (3, 12, 200, 1, 'cross'),
    (3, 12, 200, 127, 'cross'),
    (3, 12, 200, 128, 'cross'),
    (3, 12, 200, 129, 'cross'),
    (3, 12, 200, 257, 'cross'),
    (3, 16, 1, 257, 'cross'),
    (4, 12, 37, 37, 'self'),
]


def _attn_run(lib, impl, q, ldq, k, ldk, v, ldv, B, heads, Nq, Nk, scale, dev):
    D = heads * 64
    buf, out = _nan_buffer(B * Nq * D, torch.bfloat16, dev, guard=D)
    lib.d3r_set_attention_impl(impl)
    _call(lib.d3r_attention_hd64(q, ldq, k, ldk, v, ldv, _p(out), D, B, heads, Nq, Nk, scale, _lib.stream_ptr()))
    return buf, out.view(B, Nq, heads, 64).permute(0, 2, 1, 3)


@pytest.mark.timeout(600)
@pytest.mark.parametrize('regime', ['uniform', 'peaked'])
@pytest.mark.parametrize('B,heads,Nq,Nk,layout', ATTN_CASES)
def test_attention_bound_and_impl_bit_identity(cuda_device, B, heads, Nq, Nk, layout, regime):
    """d3r_attention_hd64 in the forward's layouts vs softmax(q k^T / 8) v in float64 on the same bf16 inputs; impl 2 (P through
    shared memory) and impl 3 (P in registers) give the same bits.

    Regimes: unit q, k, v (near-uniform softmax, logits ~ N(0, 1)) and q, k scaled by sqrt(6) (logits with std 6: each output
    is a few rows of V).  The kernel rounds P to bf16 before P V (the normaliser l sums the unrounded p) and O to bf16:
      elementwise  |o - ref| <= U (|ref| + Ep + Ef) + Ep + Ef,
        Ep = U min(sum_j p|v|, 8 sqrt(sum_j p^2 v^2)) / l   (rigorous, or Hoeffding at 8 sigma over the independent roundings),
        Ef = (g(Nk) + ep + 2 ds) sum_j p|v| / l + ((Nk/4 + 64) 2^-23 + ep + 2 ds) |ref|:  the P V accumulation (wgmma), the
             fp32 sum of l (Nk/4 terms per thread), ep = 2^-21 (1 + 1.5 max_j |s_j|) for ex2.approx and the rounding of its
             argument, ds = g(64) max_j (|q| |k|) / 8 for the logits' own accumulation;
      per (image, head)  |sum (o - ref) ref| <= 6 U sqrt(sum ref^4 + sum_ij (p_ij <v_j, ref_i> / l_i)^2) + sum Ef |ref|
        (Hoeffding at 6 sigma: the output and P roundings projected on ref), which resolves a common gain error of ~1 / Nk.
    Resolution: one extra zero-logit key in the ragged last block (near-uniform regime, Nk <= 257, where its weight ~1 / Nk
    is above the fp32 allowance; with logits of std 6 a logit of 0 has weight ~e^-m and the bug is harmless), and dropping
    the last key block (cases with >= 1024 query rows, so that some row draws weight from it)."""
    dev = cuda_device
    lib = _lib.get_lib()
    D = heads * 64
    scale = 0.125
    a = 1.0 if regime == 'uniform' else math.sqrt(6.0)
    seed = B * 1000 + heads * 100 + Nq + 7 * Nk + (0 if regime == 'uniform' else 50000)
    if layout == 'self':
        assert Nq == Nk
        qkv = _randn((B * Nq, 3, D), seed, dev)
        qkv[:, :2] *= a
        qkv = qkv.reshape(B * Nq, 3 * D).to(torch.bfloat16)
        qm, km, vm = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        es = qkv.element_size()
        ptrs = (qkv.data_ptr(), 3 * D, qkv.data_ptr() + D * es, 3 * D, qkv.data_ptr() + 2 * D * es, 3 * D)
    else:
        qb = (_randn((B * Nq, D), seed, dev) * a).to(torch.bfloat16)
        kv = _randn((B * Nk, 2, D), seed + 1, dev)
        kv[:, 0] *= a
        kv = kv.reshape(B * Nk, 2 * D).to(torch.bfloat16)
        qm, km, vm = qb, kv[:, :D], kv[:, D:]
        es = kv.element_size()
        ptrs = (qb.data_ptr(), D, kv.data_ptr(), 2 * D, kv.data_ptr() + D * es, 2 * D)
    try:
        buf2, out2 = _attn_run(lib, 2, *ptrs, B, heads, Nq, Nk, scale, dev)
        buf3, out3 = _attn_run(lib, 3, *ptrs, B, heads, Nq, Nk, scale, dev)
    finally:
        lib.d3r_set_attention_impl(3)
    what = f'attention {layout} B={B} heads={heads} Nq={Nq} Nk={Nk} {regime}'
    assert torch.equal(buf2.view(torch.int16), buf3.view(torch.int16)), f'{what}: impl 2 and impl 3 differ'
    assert _guard_ok(buf3, B * Nq * D), what
    out = out3

    def heads_view(t, N):
        return t.double().reshape(B, N, heads, 64).permute(0, 2, 1, 3)

    q, k, v = heads_view(qm, Nq), heads_view(km, Nk), heads_view(vm, Nk)
    s = q @ k.transpose(-1, -2) * scale
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    ref = (p @ v) / l
    pv = (p @ v.abs()) / l
    ep = U * torch.minimum(pv, 8 * torch.sqrt((p * p) @ (v * v)) / l)
    ds = _gamma(64) * (q.abs() @ k.abs().transpose(-1, -2)).amax(-1, keepdim=True) * scale
    eps_p = 2.0 ** -21 * (1 + 1.5 * s.abs().amax(-1, keepdim=True))
    ef = (_gamma(Nk) + eps_p + 2 * ds) * pv + ((Nk / 4 + 64) * 2.0 ** -23 + eps_p + 2 * ds) * ref.abs()
    e = ep + ef
    bound = U * (ref.abs() + e) + e + 1e-30
    assert torch.isfinite(out.double()).all(), f'{what}: non-finite or unwritten output'
    ratio = ((out.double() - ref).abs() / bound).max().item()
    assert ratio <= 1.0, f'{what}: elementwise worst |err|/bound = {ratio:.3f}'
    wdot = ref @ v.transpose(-1, -2)                                   # <v_j, ref_i>
    noise = (ref ** 4).sum((-1, -2)) + ((p * wdot / l) ** 2).sum((-1, -2))
    gain_bound = 6 * U * torch.sqrt(noise) + (ef * ref.abs()).sum((-1, -2)) + 1e-30

    def gain_ratio(r):
        return ((out.double() - r) * r).sum((-1, -2)).abs() / gain_bound

    gratio = gain_ratio(ref).max().item()
    assert gratio <= 1.0, f'{what}: per-head gain worst |err|/bound = {gratio:.3f}'

    def rejected(r):
        return int(((out.double() - r).abs() > bound).sum()) > 0 or bool((gain_ratio(r) > 1.0).any())

    checks = []
    if regime == 'uniform' and Nk % 128 and Nk <= 257 and B * heads * Nq >= 128:
        checks.append(('extra zero-logit key', (p @ v) / (l + torch.exp(-m))))
    if Nk > 128 and B * heads * Nq >= 1024:
        kept = 128 * ((Nk - 1) // 128)
        pk = p[..., :kept]
        checks.append(('last key block dropped', (pk @ v[..., :kept, :]) / pk.sum(-1, keepdim=True)))
    for name, bad in checks:
        assert rejected(bad), f'{what}: {name} not rejected'
    print(f'margin {what}: elementwise worst |err|/bound {ratio:.3f}, per-head gain {gratio:.3f}; rejects: '
          f'{", ".join(n for n, _ in checks) or "-"}')
