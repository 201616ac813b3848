"""The evaluation criteria on the GPU (csrc/criterion_ops.cu behind dust3r_b200.losses) against the reference's goldens, the
host port, and the host port run in float64, plus the segmented median against torch.nanmedian.

Tolerances.  The device computes every per-pixel quantity in fp32 (as the reference does) but sums in fp64 where the
reference sums in fp32 and takes the same lower medians; the remaining differences are fp32 rounding in the transform, the
normalisation and the distance, a few 1e-7 relative per value.  1e-5 relative on losses and details covers that with margin;
a wrong median, a leaked invalid pixel or a mis-ordered stage moves them by 1e-3 or more.  Against float64 the loss of a
512x384 batch of 32 pairs agrees to the same 1e-5: its fp32 inputs are exact in float64, so the difference is the device's fp32
rounding alone (and, where fp32 rounding reorders two nearly equal values, a neighbouring order statistic as median).
The median itself is compared with ==, not bit for bit: the radix order puts -0 below +0 while torch treats them as equal, so
where the two tie either may be returned."""
import copy
import math

import pytest
import torch

import dust3r_b200.losses as L
from dust3r_b200.inference import loss_of_one_batch
from dust3r_b200.utils.synth import synth_criterion_batch, synth_images

from test_criterion_host import TEST, TRAIN, check_case, close, golden, golden_cases, golden_inputs

pytestmark = pytest.mark.gpu

RTOL = 1e-5


def to(inputs, dev, dtype=None):
    return tuple({k: v.to(dev, dtype if dtype is not None and v.is_floating_point() else None) for k, v in d.items()}
                 for d in inputs)


@pytest.mark.parametrize('case', golden_cases(), ids=lambda c: c['name'])
def test_device_matches_golden_and_host(case, cuda_device, capsys):
    G = golden()
    crit = eval(case['expr'], vars(L))
    cpu = golden_inputs(G, case['inputs'])
    dev = to(cpu, cuda_device)
    before = copy.deepcopy(dev)
    loss, details = crit(*dev, **case['kwargs'])
    check_case(case, loss, details, G, rtol=RTOL)
    if case['loss'] is not None:
        assert loss.is_cuda
    host_loss, host_details = crit(*cpu, **case['kwargs'])
    check_case(dict(case, details=host_details, loss=None if isinstance(host_loss, tuple) else float(host_loss)),
               loss, details, {**{k: G[k] for k in G.files},
                               **({f'out|{case["name"]}|loss{k + 1}': host_loss[k][0].numpy() for k in range(2)}
                                  if isinstance(host_loss, tuple) else {})}, rtol=RTOL)
    for v, w in zip(dev, before):   # inputs untouched
        for k in v:
            assert torch.equal(v[k].nan_to_num(), w[k].nan_to_num()), (case['name'], k)
    if case['inputs'] == 'empty2' and case['expr'].startswith('ConfLoss'):
        assert 'NO VALID POINTS in img2' in capsys.readouterr().out


def _float64_host(expr, inputs):
    loss, details = eval(expr, vars(L))(*to(inputs, 'cpu', torch.float64))
    return float(loss), details


@pytest.mark.timeout(900)
@pytest.mark.parametrize('expr', [TRAIN, TEST])
def test_full_size_against_float64(expr, cuda_device):
    inputs = synth_criterion_batch(32, (384, 512), (384, 512), seed=21)
    ref_loss, ref_details = _float64_host(expr, inputs)
    loss, details = eval(expr, vars(L))(*to(inputs, cuda_device))
    assert close(float(loss), ref_loss, RTOL), (float(loss), ref_loss)
    assert list(details) == list(ref_details)
    for k in details:
        assert close(details[k], ref_details[k], RTOL), (k, details[k], ref_details[k])


def _median_cases(dev):
    g = torch.Generator().manual_seed(3)
    nan, inf = float('nan'), float('inf')
    yield 'odd', torch.randn(7, 101, generator=g)
    yield 'even', torch.randn(7, 100, generator=g)
    yield 'ties', torch.randint(-3, 4, (9, 64), generator=g).float()
    rows = torch.randn(6, 50, generator=g)
    rows[0] = nan            # all invalid
    rows[1, ::2] = nan       # NaN inside
    rows[2, :3] = torch.tensor([inf, -inf, inf])
    rows[3] = torch.tensor([0.0, -0.0] * 25)
    rows[4, :20] = -0.0
    rows[4, 20:40] = 0.0
    rows[5, 1:] = nan        # one value
    yield 'special', rows
    yield 'one', torch.tensor([[2.5]])
    big = torch.randn(4, 393216, generator=g)
    big[1, torch.rand(393216, generator=g) < 0.3] = nan
    big[2] = torch.round(big[2] * 4) / 4   # heavy ties across a large segment
    yield 'large', big


def test_nanmedian_matches_torch_exactly(cuda_device):
    for name, x in _median_cases(cuda_device):
        x = x.to(cuda_device)
        got = L.cuda_nanmedian(x)
        want = torch.nanmedian(x, dim=-1).values
        same = (got == want) | (got.isnan() & want.isnan())
        assert bool(same.all()), (name, got[~same], want[~same])


@pytest.mark.parametrize('expr', [TRAIN, TEST, "Regr3D(L21).with_reduction('none')"])
def test_two_calls_bit_identical(expr, cuda_device):
    inputs = to(synth_criterion_batch(4, (64, 96), (48, 64), seed=22), cuda_device)
    crit = eval(expr, vars(L))
    a, da = crit(*inputs)
    b, db = crit(*inputs)
    assert da == db or all((x == y) or (math.isnan(x) and math.isnan(y)) for x, y in zip(da.values(), db.values()))
    if isinstance(a, tuple):
        for (la, ma), (lb, mb) in zip(a, b):
            assert torch.equal(la, lb) and torch.equal(ma, mb)
    else:
        assert torch.equal(a, b)


def test_mixed_devices_raise(cuda_device):
    gt1, gt2, pred1, pred2 = synth_criterion_batch(1, (8, 12), (8, 12), seed=23)
    gt2 = {k: v.to(cuda_device) for k, v in gt2.items()}
    for expr in (TRAIN, TEST):
        with pytest.raises(ValueError, match='CUDA device'):
            eval(expr, vars(L))(gt1, gt2, pred1, pred2)


@pytest.mark.timeout(900)
def test_loss_of_one_batch_end_to_end(cuda_device):
    """A small DPT model with synthetic weights, ground truth attached to the views: loss_of_one_batch symmetrises the batch,
    runs the forward and the criterion on the device, and its result is the criterion applied to the returned predictions."""
    from test_forward_gpu import _build, _small_cfgs
    cfg, H, W = _small_cfgs()['small_dpt']
    net, _ = _build(cfg, 5, cuda_device)
    B = 2
    imgs = synth_images(2 * B, H, W, seed=4)
    gt1, gt2, _, _ = synth_criterion_batch(B, (H, W), (H, W), seed=24)
    views = []
    for k, gt in enumerate((gt1, gt2)):
        own = imgs[k * B:(k + 1) * B]
        views.append(dict(gt, img=torch.cat([x['img'] for x in own]), true_shape=torch.tensor([[H, W]] * B),
                          instance=[x['instance'] for x in own], idx=[x['idx'] for x in own]))
    crit = eval(TRAIN, vars(L))
    with torch.no_grad():
        res = loss_of_one_batch(tuple(dict(v) for v in views), net, crit, cuda_device, symmetrize_batch=True)
    loss, details = res['loss']
    assert loss.is_cuda and math.isfinite(float(loss)) and set(details) == {'conf_loss_1', 'conf_loss2', 'Regr3D_pts3d_1', 'Regr3D_pts3d_2'}
    assert res['pred1']['pts3d'].shape[0] == 2 * B
    again, again_details = crit(res['view1'], res['view2'], res['pred1'], res['pred2'])
    assert torch.equal(loss, again) and details == again_details
    with torch.no_grad():
        only = loss_of_one_batch(tuple(dict(v) for v in views), net, eval(TEST, vars(L)), cuda_device, symmetrize_batch=True,
                                 ret='loss')
    assert isinstance(only, tuple) and math.isfinite(float(only[0]))
