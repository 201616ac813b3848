"""The float64 criterion oracle (oracle/criterion_float64.py) on the CPU: it equals the host port of dust3r_b200.losses run in
float64 for every criterion family, gt_scale, norm_mode, reduction and ConfLoss, on every golden input set and on the value
and validity cases tests/test_criterion_float64_gpu.py runs; the reference's fp32 goldens lie within the bound it derives
for an fp32 evaluation; and the element-wise bounds see kernel mistakes that a 1e-5 scalar check cannot (the resolution
demonstration: a pixel dropped at a slot boundary, two compacted distances swapped across one, the upper median on an even
count, the prediction-scale clip omitted, the 1e-8 floor omitted)."""
import math

import numpy as np
import pytest
import torch

import dust3r_b200.losses as L
from dust3r_b200.utils.synth import synth_criterion_batch
from oracle import criterion_float64 as O

from test_criterion_host import golden, golden_cases, golden_inputs

KCHUNK = 4096                     # pixels of one slot of the per-pixel passes (kChunk in criterion_ops.cu)
FAMILIES = ['Regr3D', 'Regr3D_ShiftInv', 'Regr3D_ScaleInv', 'Regr3D_ScaleShiftInv']


def criterion_matrix(clip=3.0):
    """(expr, kwargs): every family x gt_scale x norm_mode x reduction, ConfLoss at alpha 0.2 and 0.5 over every family x
    gt_scale x norm_mode, and dist_clip on Regr3D with and without ConfLoss (the variants take no dist_clip)."""
    out = []
    for fam in FAMILIES:
        for gts in (False, True):
            for nm in ('avg_dis', None):
                base = f'{fam}(L21, norm_mode={nm!r}, gt_scale={gts})'
                out += [(base, {}), (base + ".with_reduction('sum')", {}), (base + ".with_reduction('none')", {})]
                out += [(f'ConfLoss({base}, alpha={a})', {}) for a in (0.2, 0.5)]
    out += [('Regr3D(L21)', dict(dist_clip=clip)), ("Regr3D(L21).with_reduction('none')", dict(dist_clip=clip)),
            ('ConfLoss(Regr3D(L21), alpha=0.2)', dict(dist_clip=clip))]
    return out


def spec(expr, kw=None):
    """(flags, reduction, dist_clip, alpha, Regr3D-family criterion) of the d3r_criterion call a criterion makes, or None for
    a combination of criteria."""
    crit = eval(expr, vars(L))
    alpha = None
    if isinstance(crit, L.ConfLoss):
        if crit._loss2 is not None or crit._alpha != 1:
            return None
        alpha, crit = crit.alpha, crit.pixel_loss
    if crit._loss2 is not None or crit._alpha != 1:
        return None
    clip = (kw or {}).get('dist_clip')
    flags = (O.NORM if crit.norm_mode else 0) | (O.GT_SCALE if crit.gt_scale else 0) | (O.SHIFT if crit._shift else 0) \
        | (O.SCALE if crit._scale else 0) | (O.CONF if alpha is not None else 0) | (O.CLIP if clip is not None else 0)
    red = 2 if alpha is not None else {'mean': 0, 'sum': 1, 'none': 2}[crit.criterion.reduction]
    return flags, red, float(clip or 0.0), float(alpha or 0.0), crit


def oracle_inputs(inputs, flags, clip, alpha, T=None, **kw):
    gt1, gt2, p1, p2 = inputs
    if T is None:
        T = torch.linalg.inv(gt1['camera_pose'].to(torch.float64))
    return O.inputs64(T, gt1['pts3d'], gt2['pts3d'], gt1['valid_mask'], gt2['valid_mask'], p1['pts3d'],
                      p2['pts3d_in_other_view'], p1['conf'], p2['conf'], flags=flags, clip=clip, alpha=alpha, **kw)


# ------------------------------------------------------------------------------------------------- value / validity cases
def add_garbage(inputs):
    """NaN, +-Inf and 1e30 in the ground truth under every invalid pixel, as synth_criterion_batch(garbage=True) puts them:
    none of it may reach a result."""
    junk = torch.tensor([float('nan'), float('inf'), -float('inf'), 1e30])
    out = tuple(dict(d) for d in inputs)
    for gt in out[:2]:
        pts = gt['pts3d'].clone()
        bad = (~gt['valid_mask'].bool()).nonzero()
        pts[bad[:, 0], bad[:, 1], bad[:, 2]] = junk[torch.arange(len(bad)) % 4, None]
        gt['pts3d'] = pts
    return out


def synth_batch(B, hw1, hw2, seed=0, garbage=True):
    """synth_criterion_batch at any view size, one-row views included: a view of fewer than two rows or columns is the
    first H * W pixels, row-major, of a two-row view."""
    src = lambda hw: hw if min(hw) >= 2 else (2, max(2, (hw[0] * hw[1] + 1) // 2))
    views = synth_criterion_batch(B, src(hw1), src(hw2), seed=seed, garbage=False)

    def crop(d, hw):
        n = hw[0] * hw[1]
        return {k: v if k == 'camera_pose' else v.reshape(B, -1, *v.shape[3:])[:, :n].reshape(B, *hw, *v.shape[3:])
                for k, v in d.items()}
    views = crop(views[0], hw1), crop(views[1], hw2), crop(views[2], hw1), crop(views[3], hw2)
    return add_garbage(views) if garbage else views


def with_masks(inputs, pattern, seed=0):
    """A batch made with garbage=False, with one of the validity patterns applied to both views' valid_mask and garbage
    under the pixels it leaves invalid."""
    gt1, gt2, p1, p2 = (dict(d) for d in inputs)
    g = torch.Generator().manual_seed(seed)
    for gt in (gt1, gt2):
        m = gt['valid_mask'].clone()
        B, H, W = m.shape
        n = H * W
        flat = m.reshape(B, n)
        if pattern == 'sparse':                     # 1 % valid
            flat &= torch.rand((B, n), generator=g) < 0.01
            flat[:, 0] = True
        elif pattern == 'slot_edges':               # only the first and last pixel of every slot
            i = torch.arange(n) % KCHUNK
            flat[:] = (i == 0) | (i == KCHUNK - 1) | (torch.arange(n) == n - 1)
        elif pattern == 'last_slot':                # only the last, partial slot
            flat[:] = torch.arange(n) >= (n - 1) // KCHUNK * KCHUNK
        elif pattern == 'pair_empty':               # pair 1 without any valid pixel, the others untouched
            flat[min(1, B - 1)] = False
        elif pattern != 'synthetic':
            raise ValueError(pattern)
        gt['valid_mask'] = flat.reshape(B, H, W)
    return add_garbage((gt1, gt2, p1, p2))


def value_case(name, B, hw1, hw2, seed=0):
    """A synthetic batch (fp32, CPU) that drives one branch of the criteria."""
    gt1, gt2, p1, p2 = synth_batch(B, hw1, hw2, seed=seed)
    if name == 'scale_tiny' or name == 'scale_huge':     # with norm_mode=None: the prediction-scale clip at 1e-3 / 1e3
        s = 1e-5 if name == 'scale_tiny' else 1e5
        p1['pts3d'] = p1['pts3d'] * s
        p2['pts3d_in_other_view'] = p2['pts3d_in_other_view'] * s
    elif name == 'zero_pred':                            # the 1e-8 floor of the normalisation factor
        p1['pts3d'] = torch.zeros_like(p1['pts3d'])
        p2['pts3d_in_other_view'] = torch.zeros_like(p2['pts3d_in_other_view'])
    elif name in ('ties', 'straddle'):                   # identity pose: the medians see the points as given
        for gt in (gt1, gt2):
            gt['camera_pose'] = torch.eye(4).expand_as(gt['camera_pose']).clone()
        pts = [gt1['pts3d'], gt2['pts3d'], p1['pts3d'], p2['pts3d_in_other_view']]
        valid = [gt1['valid_mask'], gt2['valid_mask']] * 2
        for k in range(4):
            x = pts[k].clone()
            if name == 'ties':                           # thousands of equal depths and coordinates at the median
                x = torch.round(x * 4) / 4
            else:                                        # scenes straddling x = 0 and z = 0, with exact +-0 values
                fin = x[valid[k]]
                x = x - fin.median(dim=0).values
                x[..., 0][x[..., 0].abs() < 0.05] = -0.0
                x[..., 2][x[..., 2].abs() < 0.05] = 0.0
            pts[k] = torch.where(valid[k][..., None], x, pts[k])
        gt1['pts3d'], gt2['pts3d'], p1['pts3d'], p2['pts3d_in_other_view'] = pts
    elif name == 'nan_pred':                             # one NaN at a valid pixel of pair 0, view 2
        x = p2['pts3d_in_other_view'].clone()
        nz = gt2['valid_mask'][0].nonzero()
        i, j = nz[len(nz) // 2].tolist()
        x[0, i, j, 1] = float('nan')
        p2['pts3d_in_other_view'] = x
    elif name == 'view1_empty':                          # pair 0: view 1 empty, view 2 not
        gt1 = dict(gt1)
        m = gt1['valid_mask'].clone()
        m[0] = False
        gt1['valid_mask'] = m
    elif name != 'synthetic':
        raise ValueError(name)
    return gt1, gt2, p1, p2


VALUE_CASES = ['scale_tiny', 'scale_huge', 'zero_pred', 'ties', 'straddle', 'nan_pred', 'view1_empty']


# ------------------------------------------------------------------------------------------------------ host port check
def _f64(inputs):
    return tuple({k: v.to(torch.float64) if v.is_floating_point() else v for k, v in d.items()} for d in inputs)


def _same(a, b, rtol):
    if math.isnan(b):
        return math.isnan(a)
    return a == b or abs(a - b) <= rtol * abs(b)


def check_oracle_against_host(expr, kw, inputs):
    """The oracle on float64 inputs equals the host port run in float64: losses to 1e-12 relative, per-pixel distances to
    1e-12, masks exactly, details (which the criteria return as fp32-rounded floats) to one fp32 rounding."""
    inputs = _f64(inputs)
    flags, red, clip, alpha, crit = spec(expr, kw)
    r = O.criterion64(oracle_inputs(inputs, flags, clip, alpha), red)
    loss, det = eval(expr, vars(L))(*inputs, **kw)
    name = type(crit).__name__
    want = {name + '_pts3d_1': r.out[0], name + '_pts3d_2': r.out[1]}
    if flags & O.CONF:
        want = dict(conf_loss_1=r.out[2], conf_loss2=r.out[3], **want)
    assert list(det) == list(want), expr
    for k in want:
        assert _same(det[k], want[k], 2 ** -23), (expr, k, det[k], want[k])
    if isinstance(loss, tuple):
        for v, (l, m) in enumerate(loss):
            assert torch.equal(m.reshape(m.shape[0], -1), r.valid[v]), (expr, v)
            assert l.shape == r.pix[v].shape and torch.allclose(l, r.pix[v], rtol=1e-12, atol=1e-300, equal_nan=True), (expr, v)
    else:
        assert _same(float(loss), r.out[4], 1e-12), (expr, float(loss), r.out[4])
    return r


@pytest.mark.parametrize('inputs', ['base', 'mixed', 'empty2'])
def test_oracle_matches_float64_host_port_on_golden_inputs(inputs):
    data = golden_inputs(golden(), inputs)
    for expr, kw in criterion_matrix():
        check_oracle_against_host(expr, kw, data)


@pytest.mark.parametrize('case', VALUE_CASES + ['sparse', 'slot_edges', 'last_slot', 'pair_empty'])
def test_oracle_matches_float64_host_port_on_value_cases(case):
    if case in VALUE_CASES:
        data = value_case(case, 3, (8, 12), (6, 10), seed=31)
    else:
        data = with_masks(synth_batch(3, (8, 12), (6, 10), seed=31, garbage=False), case)
    for expr, kw in criterion_matrix(clip=3.0):
        check_oracle_against_host(expr, kw, data)


def test_value_cases_reach_their_branches():
    """The value cases do what they are for: both ends of the prediction-scale clip, the 1e-8 floor, large ties at the
    median, negative and +-0 medians, a NaN that stays in its pair, a pair without valid pixels next to valid ones."""
    def run(case, expr, **kw):
        data = _f64(value_case(case, 3, (8, 12), (6, 10), seed=31)) if case in VALUE_CASES else \
            _f64(with_masks(synth_batch(3, (8, 12), (6, 10), seed=31, garbage=False), case))
        flags, red, clip, alpha, _ = spec(expr)
        return O.criterion64(oracle_inputs(data, flags, clip, alpha), red, **kw), data
    r, _ = run('scale_tiny', 'Regr3D_ScaleInv(L21, norm_mode=None)')
    assert bool((r.params['scale_pr'][0] < 1e-3).all()) and bool((r.params['scale_pr_clipped'][0] == 1e-3).all())
    r, _ = run('scale_huge', 'Regr3D_ScaleInv(L21, norm_mode=None)')
    assert bool((r.params['scale_pr'][0] > 1e3).all()) and bool((r.params['scale_pr_clipped'][0] == 1e3).all())
    r, _ = run('zero_pred', 'Regr3D(L21)')
    assert bool((r.params['nf_pr'][0] == 1e-8).all())
    r, data = run('ties', 'Regr3D_ScaleShiftInv(L21, norm_mode=None)')
    z = torch.cat([data[0]['pts3d'][..., 2][data[0]['valid_mask']], data[1]['pts3d'][..., 2][data[1]['valid_mask']]])
    assert int((z == r.params['shift_gt'][0][0]).sum()) >= 20
    r, _ = run('straddle', 'Regr3D_ScaleShiftInv(L21, norm_mode=None)')
    c = r.params['centre_gt'][0]
    assert bool((c[:, 0] <= 0).any()) and bool((c == 0).any())
    r, _ = run('nan_pred', 'Regr3D_ScaleShiftInv(L21)')
    assert math.isnan(r.out[1]) and math.isnan(r.params['nf_pr'][0][0]) and not r.params['nf_pr'][0][1:].isnan().any()
    r, _ = run('pair_empty', 'Regr3D_ScaleShiftInv(L21)')
    assert r.params['shift_gt'][0][1].isnan() and not r.params['shift_gt'][0][[0, 2]].isnan().any() and math.isfinite(r.out[4])


# -------------------------------------------------------------------------------------------------- reference goldens
def golden_oracle(case):
    """The oracle for a golden case as the reference evaluated it: fp32 inputs, fp32 sums in any order, and a pose it
    inverted in fp32 itself.  LU inversion of the 4x4 pose has a forward error of at most gamma(12) kappa(pose) |T| per
    element (Higham, backward error gamma(3n) of LU, n = 4), which enters as dT."""
    sp = spec(case['expr'], case['kwargs'])
    if sp is None:
        return None, None
    flags, red, clip, alpha, _ = sp
    data = golden_inputs(golden(), case['inputs'])
    pose = data[0]['camera_pose'].to(torch.float64)
    T = torch.linalg.inv(pose)
    kappa = float(max(np.linalg.cond(p.numpy(), np.inf) for p in pose))
    dT = O.gamma(12) * kappa * float(T.abs().max())
    return O.criterion64(oracle_inputs(data, flags, float(np.float32(clip)), float(np.float32(alpha)), T=T, dT=dT,
                                       fp32_sums=True), red), sp


@pytest.mark.parametrize('case', golden_cases(), ids=lambda c: c['name'])
def test_reference_golden_within_oracle_bound(case):
    r, sp = golden_oracle(case)
    if r is None:
        pytest.skip('a combination of criteria: no single d3r_criterion call')
    G = golden()
    flags, red, _, _, crit = sp
    name = type(crit).__name__
    want = {name + '_pts3d_1': 0, name + '_pts3d_2': 1}
    if flags & O.CONF:
        want = dict(conf_loss_1=2, conf_loss2=3, **want)
    worst = 0.0
    for k, i in want.items():
        got = case['details'][k]
        assert math.isnan(got) == math.isnan(r.out[i]), k
        worst = max(worst, O.ratio(abs(got - r.out[i]), r.dout[i]))
    if case['loss'] is not None:
        worst = max(worst, O.ratio(abs(case['loss'] - r.out[4]), r.dout[4]))
    else:
        for v in range(2):
            m = G[f'out|{case["name"]}|mask{v + 1}']
            assert np.array_equal(m.reshape(m.shape[0], -1), r.valid[v].numpy())
            worst = max(worst, O.ratio((torch.from_numpy(G[f'out|{case["name"]}|loss{v + 1}']).double() - r.pix[v]).abs(), r.dpix[v]))
    print(case['name'], 'worst err/bound', worst)
    assert worst <= 1, worst


# ---------------------------------------------------------------------------------------------- resolution demonstration
def _rel(a, b):
    return abs(a - b) / abs(b)


def _fca(expr):
    flags, _, clip, alpha, _ = spec(expr)
    return flags, clip, alpha


def resolution_demo():
    """Each kernel mistake built on the float64 side: (worst err / element-wise bound, relative change of the scalar loss).
    The slot-boundary mistakes use two pairs of 384x512 + 288x512 (48 and 36 full slots, about 0.6 M valid pixels a view)."""
    demo = {}
    big = _f64(synth_criterion_batch(2, (384, 512), (288, 512), seed=41))
    flags, red, clip, alpha, _ = spec("Regr3D_ScaleShiftInv(L21).with_reduction('none')")
    inp = oracle_inputs(big, flags, clip, alpha)
    r = O.criterion64(inp, red)
    tight = O.criterion64(inp, red, P=O.params_tensor(r, inp.B))   # the per-pixel bound the GPU test uses
    pix, dpix = tight.pix[0], tight.dpix[0]
    n1 = big[0]['valid_mask'][0].numel()
    mean = lambda x: float(x.mean())
    # 1. the first valid pixel of the second slot of pair 1, view 1 dropped: its mask bit flips, the compaction shifts
    flat = r.valid[0].reshape(-1)
    drop = n1 + KCHUNK + int(flat[n1 + KCHUNK:].nonzero()[0])
    k = int(flat[:drop].sum())
    bad = torch.cat([pix[:k], pix[k + 1:]])
    demo['dropped pixel'] = (O.ratio((bad - pix[:-1]).abs(), dpix[:-1]), _rel(mean(bad), mean(pix)))
    # 2. the last distance of slot 0 and the first of slot 1 of pair 0, view 1 swapped
    k = int(flat[:KCHUNK].sum())
    bad = pix.clone()
    bad[k - 1], bad[k] = pix[k], pix[k - 1]
    demo['swapped across a slot'] = (O.ratio((bad - pix).abs(), dpix), _rel(mean(bad), mean(pix)))
    # 3. rank n / 2 instead of (n - 1) / 2 on an even count (a small batch, where neighbouring order statistics differ)
    small = _f64(synth_criterion_batch(3, (37, 53), (37, 53), seed=42))
    inp = oracle_inputs(small, *_fca("Regr3D_ScaleShiftInv(L21)"))
    good, upper = O.criterion64(inp, 0), O.criterion64(inp, 0, upper_median=True)
    even = sum(m.sum(1) for m in good.valid) % 2 == 0
    assert bool(even.any())
    v, e = good.params['shift_gt']
    demo['upper median'] = (O.ratio((upper.params['shift_gt'][0] - v).abs()[even], e[even]), _rel(upper.out[4], good.out[4]))
    # 4. the prediction-scale clip omitted, 5. the 1e-8 floor omitted
    for name, case, expr, kw in (('no scale clip', 'scale_tiny', 'Regr3D_ScaleInv(L21, norm_mode=None)', dict(scale_clip=False)),
                                 ('no 1e-8 floor', 'zero_pred', 'Regr3D(L21)', dict(nf_floor=False))):
        data = _f64(value_case(case, 3, (37, 53), (37, 53), seed=43))
        inp = oracle_inputs(data, *_fca(expr))
        good, bad = O.criterion64(inp, 0), O.criterion64(inp, 0, **kw)
        r_ = math.inf if math.isnan(bad.out[4]) else O.ratio(abs(bad.out[4] - good.out[4]), good.dout[4])
        demo[name] = (r_, math.inf if math.isnan(bad.out[4]) else _rel(bad.out[4], good.out[4]))
    return demo


@pytest.mark.timeout(600)
def test_resolution_demonstration():
    """Every mistake exceeds the element-wise bound; the two slot-boundary mistakes stay inside the 1e-5 relative scalar
    tolerance of tests/test_criterion_gpu.py, so only the element-wise checks can see them."""
    demo = resolution_demo()
    for name, (r, rel) in demo.items():
        print(f'{name:24s} err/bound {r:10.3g}   scalar change {rel:9.3g} ({"inside" if rel <= 1e-5 else "outside"} 1e-5)')
    for name, (r, rel) in demo.items():
        assert r > 1, (name, r)
    assert demo['dropped pixel'][1] <= 1e-5 and demo['swapped across a slot'][1] <= 1e-5
