"""d3r_criterion and d3r_segmented_nanmedian (csrc/criterion_ops.cu) element by element against the float64 oracle
(oracle/criterion_float64.py), at the shapes where the slot tiling of the per-pixel passes (kChunk = 4096 pixels) can go
wrong: one pixel, one slot less one, exactly one slot, one slot plus one, ragged multi-slot views of different sizes, a
pair of 1 + 8193 pixels, and 257 pairs.

The kernel is called through ctypes with buffers the test allocates, so the test knows the exact fp32 T the kernel read
and reads the per-pair stage parameters back from the workspace: its first kFields * B floats, field-major, in the order
of `enum Field`.  Per case it compares
  - the stage parameters (normalisation factors, depth shifts, centres, scales) with the float64 pipeline, within the
    largest element bound of their column (the medians) or the bound of the sums (the normalisation factors);
  - every mask bit exactly (pixels within rounding of dist_clip are settled by the device's bit and counted);
  - every compacted per-pixel distance with the float64 loss pass fed the device's own parameters (a bound that does not
    depend on which tied element a median picked);
  - the valid counts out[5..6] exactly, and out[0..4] with both the end-to-end bound (float64 parameters) and the bound
    of the loss pass fed the device's parameters;
  - NaN or +-Inf where the float64 pipeline has one, and nowhere else.
Every call also checks that the kernel stays inside its buffers: a guard region after the queried workspace size keeps
its byte pattern, the per-pixel outputs keep their sentinel from the valid count onwards, out[7] is untouched, every mask
byte is 0 or 1 and the inputs are unchanged.

Every bound constant is derived in oracle/criterion_float64.py; none is fitted.  Worst err / bound observed on an H100
80GB HBM3 (700 W), over the whole file (printed at the end of the module):
    stage parameters   nf_gt 0.149  nf_pr 0.507  shift_gt 0.313  shift_pr 0.431  centre_gt 0.286  centre_pr 0.511
                       scale_gt 0.090  scale_pr 0.217
    per-pixel distance 0.62 (device parameters)
    out[0..4]          end to end 0.082 / 0.143 / 0.085 / 0.061 / 0.105;  device parameters 0.111 / 0.143 / 0.085 /
                       0.064 / 0.119
    mask bits within rounding of dist_clip: at most 222 in one call (the quantised 'ties' case, where many |g| are
                       exactly 3); every other bit matched exactly.
Argument limits, with buffers of the real size: 10922 pairs of 1 + 1 pixels run and 10923 raise (6 B <= 65535, the grid
of the centre medians); d3r_segmented_nanmedian runs 65535 rows and raises at 65536.  seg_len >= 2^32 and
B (n1 + n2) >= 2^31 are left untested: real buffers for them take 16 GB or more."""
from collections import defaultdict

import numpy as np
import pytest
import torch

import dust3r_b200.losses as L
from dust3r_b200 import _lib
from oracle import criterion_float64 as O

from test_criterion_float64_host import VALUE_CASES, criterion_matrix, spec, synth_batch, value_case, with_masks
from test_criterion_host import TEST, TRAIN

pytestmark = pytest.mark.gpu

GUARD = 4096
SENTINEL = -7.25            # the per-pixel outputs and out[] before the call
WORST = defaultdict(float)


@pytest.fixture(scope='module', autouse=True)
def report_worst():
    yield
    print('\nworst err / bound:')
    for k, v in sorted(WORST.items()):
        print(f'  {k:28s} {v:.3g}')


def _bits(t):
    return t.contiguous().view(torch.uint8).clone()


def device_call(inputs, flags, red, clip, alpha, dev):
    """One d3r_criterion call on caller-allocated buffers: (T, P (kFields, B), out, per-pixel distances [:count], masks),
    after the buffer checks listed in the module docstring."""
    gt1, gt2, p1, p2 = inputs
    B = gt1['pts3d'].shape[0]
    n1, n2 = gt1['valid_mask'][0].numel(), gt2['valid_mask'][0].numel()
    T = torch.linalg.inv(gt1['camera_pose'].to(torch.float64)).float().contiguous()
    f32 = lambda t: t.to(dev, torch.float32).contiguous()
    u8 = lambda m: (m != 0).to(dev, torch.uint8).contiguous()
    ins = [f32(T), f32(gt1['pts3d']), f32(gt2['pts3d']), u8(gt1['valid_mask']), u8(gt2['valid_mask']), f32(p1['pts3d']),
           f32(p2['pts3d_in_other_view']), f32(p1['conf']), f32(p2['conf'])]
    before = [_bits(t) for t in ins]
    lib = _lib.get_lib()
    nbytes = int(lib.d3r_criterion_workspace_bytes(B, n1, n2, flags))
    ws = torch.full((nbytes + GUARD,), 0xA5, dtype=torch.uint8, device=dev)
    out = torch.full((8,), SENTINEL, device=dev)
    pixels = red == 2
    pix = [torch.full((B * n,), SENTINEL, device=dev) for n in (n1, n2)] if pixels else [None, None]
    msk = [torch.full((B * n,), 7, dtype=torch.uint8, device=dev) for n in (n1, n2)]
    ptr = lambda t: None if t is None else t.data_ptr()
    conf = ins[7:] if flags & O.CONF else [None, None]
    _lib.check(lib.d3r_criterion(B, n1, n2, flags, red, clip, alpha, *map(ptr, ins[:7] + conf), out.data_ptr(),
                                 ptr(pix[0]), ptr(pix[1]), msk[0].data_ptr(), msk[1].data_ptr(), ws.data_ptr(), nbytes,
                                 torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize(dev)
    assert bool((ws[nbytes:] == 0xA5).all()), 'write past the workspace size'
    assert float(out[7]) == SENTINEL, 'out[7] written'
    for t, b in zip(ins, before):
        assert torch.equal(_bits(t), b), 'input modified'
    cnt = out[5:7].view(torch.int32).tolist()
    for m in msk:
        assert bool((m <= 1).all()), 'mask byte not written or not 0/1'
    if pixels:
        for v in range(2):
            assert bool((pix[v][cnt[v]:] == SENTINEL).all()), 'per-pixel output written past the valid count'
    P = ws[:4 * O.K_FIELDS * B].view(torch.float32).reshape(O.K_FIELDS, B).cpu()
    return dict(T=T, P=P, out=out.cpu(), cnt=cnt, pix=[None if p is None else p[:c].cpu() for p, c in zip(pix, cnt)],
                msk=[m.cpu().reshape(B, -1) != 0 for m in msk], ws=ws[:nbytes])


def _cmp(name, dev, ref, bound):
    """err / bound of the finite values; the device is non-finite exactly where the float64 value is.  NaN and +-Inf count
    as one class: a pair whose scale is 0 (one valid point, or two that tie) divides by zero, and whether 0 / 0 or x / 0
    results turns on an exact fp32 cancellation the float64 pass does not reproduce."""
    dev, ref, bound = (torch.as_tensor(x, dtype=torch.float64).reshape(-1) for x in (dev, ref, bound))
    assert torch.equal(dev.isfinite(), ref.isfinite()), (name, 'non-finite pattern', dev, ref)
    ok = ref.isfinite()
    err = torch.where(dev[ok] == ref[ok], torch.zeros_like(dev[ok]), (dev[ok] - ref[ok]).abs())
    r = O.ratio(err, bound[ok])
    WORST[name] = max(WORST[name], r)
    assert r <= 1, (name, r)
    return r


def check(inputs, expr, kw, dev, label=''):
    """The comparisons of the module docstring for one criterion on one batch; returns the device result."""
    flags, red, clip, alpha, _ = spec(expr, kw)
    clip32, alpha32 = float(np.float32(clip)), float(np.float32(alpha))
    d = device_call(inputs, flags, red, clip32, alpha32, dev)
    gt1, gt2, p1, p2 = inputs
    inp = O.inputs64(d['T'], gt1['pts3d'], gt2['pts3d'], gt1['valid_mask'], gt2['valid_mask'], p1['pts3d'],
                     p2['pts3d_in_other_view'], p1['conf'], p2['conf'], flags=flags, clip=clip32, alpha=alpha32)
    r64 = O.criterion64(inp, red, decide=d['msk'])
    rdev = O.criterion64(inp, red, P=d['P'], decide=d['msk'])
    where = f'{label} {expr} {kw}'
    for v in range(2):
        und = r64.undecided[v]
        assert torch.equal(d['msk'][v][~und], r64.valid[v][~und]), (where, 'mask', v)
        WORST['undecided mask bits'] = max(WORST['undecided mask bits'], int(und.sum()))
    assert d['cnt'] == r64.count, (where, d['cnt'], r64.count)
    fields = ['nf_gt', 'nf_pr'] + (['shift_gt', 'shift_pr'] if flags & O.SHIFT else []) \
        + (['centre_gt', 'centre_pr', 'scale_gt', 'scale_pr'] if flags & O.SCALE else [])
    Pdev = d['P'].to(torch.float64)
    for name in fields:
        val, bnd = r64.params[name]
        i = O.FIELDS.index(name + '_x' if name.startswith('centre') else name)
        _cmp(f'param {name}', Pdev[i:i + 3].T if name.startswith('centre') else Pdev[i], val, bnd)
    if red == 2:
        for v in range(2):
            _cmp('pixel distance', d['pix'][v], rdev.pix[v], rdev.dpix[v])
    out = d['out'][:5].tolist()
    for k in range(5):
        _cmp(f'out[{k}] end to end', out[k], r64.out[k], r64.dout[k])
        _cmp(f'out[{k}] device params', out[k], rdev.out[k], rdev.dout[k])
    return d


# ------------------------------------------------------------------------------------------------------------ shapes
SHAPES = {
    '1x1_B3': ((1, 1), (1, 1), 3),
    '1x4095_B3': ((1, 4095), (1, 4095), 3),
    '1x4096_B1': ((1, 4096), (1, 4096), 1),
    '1x4097_B3': ((1, 4097), (1, 4097), 3),
    '3x2731_B1': ((3, 2731), (3, 2731), 1),
    '37x53_B33': ((37, 53), (37, 53), 33),
    '1+8193_B3': ((1, 1), (3, 2731), 3),
    '224x224_B3': ((224, 224), (224, 224), 3),
    '16x16_B257': ((16, 16), (16, 16), 257),
}


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('shape', list(SHAPES))
def test_full_criterion_matrix_at_ragged_shapes(shape, cuda_device):
    hw1, hw2, B = SHAPES[shape]
    inputs = synth_batch(B, hw1, hw2, seed=51)
    for expr, kw in criterion_matrix(clip=3.0):
        check(inputs, expr, kw, cuda_device, shape)


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('expr', [TRAIN, TEST, "Regr3D_ScaleShiftInv(L21, gt_scale=True).with_reduction('none')"])
def test_full_size(expr, cuda_device):
    """32 pairs of 384x512 + 288x512 (48 and 36 slots per view)."""
    check(synth_batch(32, (384, 512), (288, 512), seed=52), expr, {}, cuda_device, 'full size')


@pytest.mark.timeout(1200)
def test_portrait_against_landscape(cuda_device):
    inputs = synth_batch(3, (512, 384), (384, 512), seed=53)
    for expr in (TRAIN, TEST, "Regr3D_ScaleShiftInv(L21).with_reduction('none')", "Regr3D(L21, norm_mode=None).with_reduction('none')"):
        check(inputs, expr, {}, cuda_device, 'portrait')


PATTERN_EXPRS = [TRAIN, TEST, "Regr3D(L21).with_reduction('none')", "Regr3D_ScaleShiftInv(L21).with_reduction('none')",
                 "Regr3D_ShiftInv(L21).with_reduction('sum')", "Regr3D_ScaleInv(L21, gt_scale=True).with_reduction('none')",
                 "ConfLoss(Regr3D_ScaleShiftInv(L21, norm_mode=None), alpha=0.5)"]


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('pattern', ['synthetic', 'sparse', 'slot_edges', 'last_slot', 'pair_empty', 'view1_empty'])
def test_validity_patterns(pattern, cuda_device):
    """Ragged multi-slot views (8193 = 2 slots + 1 pixel, and 4097 pixels); a pair without valid pixels must leave the
    others' medians alone, and an empty view 1 next to a full view 2 must not reach other pairs."""
    if pattern == 'view1_empty':
        inputs = value_case('view1_empty', 3, (3, 2731), (1, 4097), seed=54)
    else:
        inputs = with_masks(synth_batch(3, (3, 2731), (1, 4097), seed=54, garbage=False), pattern)
    for expr in PATTERN_EXPRS:
        check(inputs, expr, {}, cuda_device, pattern)


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('case', VALUE_CASES)
def test_value_cases(case, cuda_device):
    """Both ends of the prediction-scale clip, the 1e-8 floor, ties at the median, negative and +-0 medians, a NaN at a
    valid prediction (NaN exactly where the float64 pipeline, and the host port, have it) and an empty view 1."""
    inputs = value_case(case, 3, (3, 2731), (1, 4097), seed=55)
    for expr, kw in criterion_matrix(clip=3.0):
        check(inputs, expr, kw, cuda_device, case)
    if case == 'nan_pred':
        host = L.Regr3D_ScaleShiftInv(L.L21).with_reduction('none')
        (hl1, _), (hl2, _) = host(*inputs)[0]
        dev_in = tuple({k: v.to(cuda_device) for k, v in x.items()} for x in inputs)
        (dl1, _), (dl2, _) = host(*dev_in)[0]
        for h, g in ((hl1, dl1), (hl2, dl2)):
            assert torch.equal(h.isnan(), g.cpu().isnan())


def test_two_calls_bit_identical(cuda_device):
    inputs = synth_batch(3, (3, 2731), (37, 53), seed=56)
    flags, red, clip, alpha, _ = spec("Regr3D_ScaleShiftInv(L21).with_reduction('none')")
    a = device_call(inputs, flags, red, clip, alpha, cuda_device)
    b = device_call(inputs, flags, red, clip, alpha, cuda_device)
    for k in ('P', 'out'):
        assert torch.equal(_bits(a[k]), _bits(b[k])), k
    for v in range(2):
        assert torch.equal(_bits(a['pix'][v]), _bits(b['pix'][v])) and torch.equal(a['msk'][v], b['msk'][v])


# ---------------------------------------------------------------------------------------------------- argument limits
@pytest.mark.timeout(600)
def test_pair_count_limit(cuda_device):
    """6 B <= 65535: 10922 pairs of 1 + 1 pixels run (and match the oracle), 10923 raise."""
    inputs = synth_batch(10922, (1, 1), (1, 1), seed=57)
    check(inputs, TEST, {}, cuda_device, 'B=10922')
    check(inputs, "Regr3D_ScaleShiftInv(L21).with_reduction('none')", {}, cuda_device, 'B=10922')
    more = synth_batch(10923, (1, 1), (1, 1), seed=57)
    flags, red, clip, alpha, _ = spec(TEST)
    with pytest.raises(_lib.D3RError, match='supported range'):
        device_call(more, flags, red, clip, alpha, cuda_device)


def test_median_row_count_limit(cuda_device):
    """n_seg <= 65535 (the grid's y extent): 65535 rows run and equal torch.nanmedian, 65536 raise."""
    g = torch.Generator().manual_seed(58)
    x = torch.randn(65535, 3, generator=g).to(cuda_device)
    assert _same_median(L.cuda_nanmedian(x), torch.nanmedian(x, dim=-1).values)
    with pytest.raises(_lib.D3RError, match='n_seg'):
        L.cuda_nanmedian(torch.zeros(65536, 1, device=cuda_device))


# -------------------------------------------------------------------------------------------------------- nanmedian
def _same_median(got, want):
    return bool(((got == want) | (got.isnan() & want.isnan())).all())


def _median_rows():
    g = torch.Generator().manual_seed(59)
    nan, inf = float('nan'), float('inf')
    for n in (4095, 4096, 4097, 8193):
        yield f'len {n}', torch.randn(5, n, generator=g)
        x = torch.randn(5, n, generator=g)
        x[:, 0 if n % 2 == 0 else -1] = nan     # one NaN flips the parity of the count
        yield f'len {n}, one NaN', x
    # non-NaN values that share their top 24 bits: the last 8-bit digit decides
    base = torch.tensor([1.2345], dtype=torch.float32).view(torch.int32)
    for n in (4097, 8193):
        bits = (base & ~0xff) | torch.randint(0, 256, (4, n), generator=g, dtype=torch.int32)
        x = bits.view(torch.float32)
        x[1] = -x[1]
        x[2, ::3] = nan
        yield f'top 24 bits shared, len {n}', x
    # denormals with +-0 and +-Inf
    x = torch.empty(6, 4097)
    for r in range(6):
        d = (torch.randint(-(1 << 23) + 1, 1 << 23, (4097,), generator=g, dtype=torch.int32)).abs().view(torch.float32)
        sign = torch.where(torch.rand(4097, generator=g) < 0.5, -1.0, 1.0)
        x[r] = d * sign
        k = torch.randperm(4097, generator=g)
        x[r, k[:300]] = 0.0
        x[r, k[300:600]] = -0.0
        x[r, k[600:610]] = inf
        x[r, k[610:615 + r]] = -inf
    assert bool((x[x.abs() < 1.2e-38] != 0).any())
    yield 'denormals, +-0, +-Inf', x
    # a single non-NaN value at the last position of a multi-chunk row
    for n in (4097, 8193, 12288):
        x = torch.full((3, n), nan)
        x[:, -1] = torch.tensor([-3.5, 0.0, 7.25])
        yield f'one value last, len {n}', x


def test_nanmedian_edges_match_torch_exactly(cuda_device):
    for name, x in _median_rows():
        x = x.to(cuda_device)
        got, want = L.cuda_nanmedian(x), torch.nanmedian(x, dim=-1).values
        assert _same_median(got, want), (name, got, want)
