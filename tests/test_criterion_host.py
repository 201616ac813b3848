"""The host port of the evaluation criteria (dust3r_b200.losses on CPU tensors) against the unmodified reference's
dust3r/losses.py, through tests/golden/criterion.npz (tests/golden/make_criterion_golden.py), and, when DUST3R_REFERENCE
points at a reference checkout, against the live classes.

Tolerance: the host port restates the reference's fp32 torch code; its geotrf multiplies by the transposed matrix where the
reference uses einsum, so the points differ in the last bits and the losses to a few 1e-7 relative.  2e-6 relative leaves
room for that and nothing else."""
import builtins
import copy
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN

import dust3r_b200.losses as L
from dust3r_b200.inference import loss_of_one_batch
from dust3r_b200.utils.synth import synth_criterion_batch

RTOL = 2e-6
TRAIN = "ConfLoss(Regr3D(L21, norm_mode='avg_dis'), alpha=0.2)"
TEST = "Regr3D_ScaleShiftInv(L21, gt_scale=True)"


def golden():
    return np.load(os.path.join(GOLDEN, 'criterion.npz'))


def golden_inputs(G, name):
    return tuple({key.split('|')[3]: torch.from_numpy(G[key].copy()) for key in G.files if key.startswith(f'in|{name}|{k}|')}
                 for k in range(4))


def golden_cases():
    return json.loads(str(golden()['meta']))


def close(a, b, rtol=RTOL):
    if math.isnan(b):
        return math.isnan(a)
    return abs(a - b) <= rtol * max(abs(b), 1e-6)


def check_case(case, loss, details, G, rtol=RTOL):
    name = case['name']
    assert list(details) == list(case['details']), name
    for k, v in case['details'].items():
        assert isinstance(details[k], float), (name, k)
        assert close(details[k], v, rtol), (name, k, details[k], v)
    if case['loss'] is None:
        for k, (lk, mk) in enumerate(loss):
            ref_l, ref_m = G[f'out|{name}|loss{k + 1}'], G[f'out|{name}|mask{k + 1}']
            assert mk.dtype == torch.bool and np.array_equal(mk.cpu().numpy(), ref_m), name
            assert lk.shape == ref_l.shape, name
            np.testing.assert_allclose(lk.cpu().numpy(), ref_l, rtol=rtol * 10, atol=1e-6, err_msg=name)
    else:
        assert torch.is_tensor(loss) and loss.ndim == 0 and not loss.requires_grad, name
        assert close(float(loss), case['loss'], rtol), (name, float(loss), case['loss'])


@pytest.mark.parametrize('case', golden_cases(), ids=lambda c: c['name'])
def test_host_port_matches_reference_golden(case, capsys):
    G = golden()
    crit = eval(case['expr'], vars(L))
    assert repr(crit) == case['repr']
    loss, details = crit(*golden_inputs(G, case['inputs']), **case['kwargs'])
    check_case(case, loss, details, G)
    if case['inputs'] == 'empty2' and case['expr'].startswith('ConfLoss'):
        assert 'NO VALID POINTS in img2' in capsys.readouterr().out


@pytest.mark.skipif(not os.environ.get('DUST3R_REFERENCE'), reason='DUST3R_REFERENCE not set')
@pytest.mark.parametrize('case', golden_cases(), ids=lambda c: c['name'])
def test_host_port_matches_live_reference(case):
    sys.path.insert(0, os.environ['DUST3R_REFERENCE'])
    import dust3r.losses as ref
    G = golden()
    inputs = golden_inputs(G, case['inputs'])
    plain_print = builtins.print
    builtins.print = lambda *a, force=False, **kw: plain_print(*a, **kw)
    try:
        rc = eval(case['expr'], vars(ref))
        rloss, rdetails = rc(*copy.deepcopy(inputs), **case['kwargs'])
    finally:
        builtins.print = plain_print
    crit = eval(case['expr'], vars(L))
    assert repr(crit) == repr(rc) and crit.get_name() == rc.get_name()
    live = dict(case, repr=repr(rc), details=rdetails, loss=None if isinstance(rloss, tuple) else float(rloss))
    for k in range(2):
        if isinstance(rloss, tuple):
            G = dict(G)
            G[f'out|{case["name"]}|loss{k + 1}'] = rloss[k][0].numpy()
            G[f'out|{case["name"]}|mask{k + 1}'] = rloss[k][1].numpy()
    loss, details = crit(*inputs, **case['kwargs'])
    check_case(live, loss, details, G)


def test_readme_strings_eval_in_module():
    train, test = eval(TRAIN, vars(L)), eval(TEST, vars(L))
    assert isinstance(train, torch.nn.Module) and isinstance(test, torch.nn.Module)
    assert repr(train) == 'ConfLoss(Regr3D(L21Loss()))' and train.pixel_loss.criterion.reduction == 'none'
    assert repr(test) == 'Regr3D_ScaleShiftInv(L21Loss())'
    assert train.to('cpu') is train
    assert [c.__name__ for c in type(test).__mro__[:4]] == ['Regr3D_ScaleShiftInv', 'Regr3D_ScaleInv', 'Regr3D_ShiftInv', 'Regr3D']


def test_algebra_names_and_reduction():
    a, b = eval('Regr3D(L21)', vars(L)), eval(TEST, vars(L))
    combo = 2 * a + b
    assert repr(combo) == '2*Regr3D(L21Loss()) + Regr3D_ScaleShiftInv(L21Loss())'
    none = a.with_reduction('none')
    assert none.criterion.reduction == 'none' and a.criterion.reduction == 'mean'
    inputs = synth_criterion_batch(2, (8, 12), (8, 12), seed=5)
    lc, dc = combo(*inputs)
    la, da = a(*inputs)
    lb, db = b(*inputs)
    assert close(float(lc), 2 * float(la) + float(lb), 1e-6)
    assert dc == da | db


@pytest.mark.parametrize('expr', [TRAIN, TEST, "Regr3D_ScaleShiftInv(L21, norm_mode=None)",
                                  "ConfLoss(Regr3D_ScaleInv(L21, norm_mode=None), alpha=0.3)"])
def test_inputs_are_not_modified(expr):
    inputs = synth_criterion_batch(2, (8, 12), (6, 10), seed=6)
    before = copy.deepcopy(inputs)
    eval(expr, vars(L))(*inputs)
    for v, w in zip(inputs, before):
        assert v.keys() == w.keys()
        for k in v:
            assert torch.equal(v[k].nan_to_num(), w[k].nan_to_num()), (expr, k)


def test_empty_view_does_not_crash(capsys):
    inputs = synth_criterion_batch(2, (8, 12), (8, 12), seed=7, empty_view2=True)
    loss, details = eval(TRAIN, vars(L))(*inputs)
    assert 'NO VALID POINTS in img2' in capsys.readouterr().out
    assert details['conf_loss2'] == 0.0 and math.isnan(details['Regr3D_pts3d_2'])
    assert close(float(loss), details['conf_loss_1'], 1e-7)


def test_no_autograd_graph():
    gt1, gt2, pred1, pred2 = synth_criterion_batch(1, (8, 12), (8, 12), seed=8)
    pred1['pts3d'].requires_grad_(True)
    loss, _ = eval(TRAIN, vars(L))(gt1, gt2, pred1, pred2)
    assert not loss.requires_grad and loss.grad_fn is None


def test_uint8_mask_counts_as_bool():
    inputs = synth_criterion_batch(2, (8, 12), (8, 12), seed=9, garbage=False)
    l_bool, d_bool = eval(TEST, vars(L))(*inputs)
    for v in inputs[:2]:
        v['valid_mask'] = v['valid_mask'].to(torch.uint8)
    l_u8, d_u8 = eval(TEST, vars(L))(*inputs)
    assert float(l_bool) == float(l_u8) and d_bool == d_u8


@pytest.mark.parametrize('mode', ['avg_log1p', 'avg_warp-log1p', 'median_dis', 'sqrt_dis'])
def test_unsupported_norm_modes_raise(mode):
    with pytest.raises(NotImplementedError, match='avg_dis'):
        L.Regr3D(L.L21, norm_mode=mode)
    with pytest.raises(NotImplementedError, match='avg_dis'):
        L.normalize_pointcloud(torch.zeros(1, 2, 2, 3), None, mode)


def test_variants_take_no_dist_clip():
    inputs = synth_criterion_batch(1, (8, 12), (8, 12), seed=10)
    with pytest.raises(TypeError):
        eval(TEST, vars(L))(*inputs, dist_clip=2.0)


class _StandIn(torch.nn.Module):
    """A model returning fixed predictions for the (symmetrised) batch, recording what it was called with."""

    def __init__(self, pred1, pred2):
        super().__init__()
        self.pred1, self.pred2, self.calls = pred1, pred2, []

    def forward(self, view1, view2):
        self.calls.append((view1, view2))
        return dict(self.pred1), dict(self.pred2)


def test_loss_of_one_batch_with_criterion():
    gt1, gt2, pred1, pred2 = synth_criterion_batch(2, (8, 12), (8, 12), seed=11)
    from dust3r_b200.inference import make_batch_symmetric
    sym1, sym2 = make_batch_symmetric((dict(gt1), dict(gt2)))
    # predictions for the symmetrised batch (4 pairs)
    p1 = {k: torch.cat([v, v]) for k, v in pred1.items()}
    p2 = {k: torch.cat([v, v]) for k, v in pred2.items()}
    model = _StandIn(p1, p2)
    crit = eval(TEST, vars(L))
    res = loss_of_one_batch((dict(gt1), dict(gt2)), model, crit, 'cpu', symmetrize_batch=True)
    assert set(res) == {'view1', 'view2', 'pred1', 'pred2', 'loss'}
    assert torch.equal(model.calls[0][0]['pts3d'].nan_to_num(), sym1['pts3d'].nan_to_num())
    loss, details = res['loss']
    ref_loss, ref_details = crit(res['view1'], res['view2'], res['pred1'], res['pred2'])
    assert float(loss) == float(ref_loss) and details == ref_details
    only = loss_of_one_batch((dict(gt1), dict(gt2)), _StandIn(pred1, pred2), crit, 'cpu', ret='loss')
    assert isinstance(only, tuple) and len(only) == 2 and set(only[1]) == set(details)
