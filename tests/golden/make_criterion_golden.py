"""Generates tests/golden/criterion.npz: what the UNMODIFIED reference's dust3r/losses.py returns, on CPU in fp32, for the
evaluation criteria that tests/test_criterion_host.py and tests/test_criterion_gpu.py check dust3r_b200.losses against.

    DUST3R_REFERENCE=<path to a naver/dust3r checkout> python tests/golden/make_criterion_golden.py

Inputs (dust3r_b200.utils.synth.synth_criterion_batch, stored in the fixture) and cases are listed in CASES; each case stores
the criterion's repr, its loss (float, or the per-pixel losses and masks with reduction 'none') and its detail dict.
The reference's ConfLoss calls print(..., force=True), which only its training process accepts: the builtin print is wrapped
to take that keyword while the cases run.
"""
import builtins
import copy
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from dust3r_b200.utils.synth import synth_criterion_batch  # noqa: E402

TRAIN = "ConfLoss(Regr3D(L21, norm_mode='avg_dis'), alpha=0.2)"
TEST = "Regr3D_ScaleShiftInv(L21, gt_scale=True)"

# input set -> synth_criterion_batch arguments
INPUTS = {
    'base': dict(B=3, hw1=(32, 48), hw2=(32, 48), seed=1),                      # NaN / Inf / 1e30 under the invalid pixels
    'mixed': dict(B=2, hw1=(32, 48), hw2=(24, 40), seed=2),                     # views of different sizes
    'empty2': dict(B=2, hw1=(16, 24), hw2=(16, 24), seed=3, empty_view2=True),  # no valid pixel in view 2
}

# (name, criterion expression, input set, keyword arguments of the call)
CASES = [
    ('train', TRAIN, 'base', {}),
    ('test', TEST, 'base', {}),
    ('regr3d', 'Regr3D(L21)', 'base', {}),
    ('regr3d_gts', 'Regr3D(L21, gt_scale=True)', 'base', {}),
    ('shift', 'Regr3D_ShiftInv(L21)', 'base', {}),
    ('shift_gts', 'Regr3D_ShiftInv(L21, gt_scale=True)', 'base', {}),
    ('scale', 'Regr3D_ScaleInv(L21)', 'base', {}),
    ('scale_gts', 'Regr3D_ScaleInv(L21, gt_scale=True)', 'base', {}),
    ('scaleshift', 'Regr3D_ScaleShiftInv(L21)', 'base', {}),
    ('nonorm', 'Regr3D(L21, norm_mode=None)', 'base', {}),
    ('nonorm_scaleshift', 'Regr3D_ScaleShiftInv(L21, norm_mode=None)', 'base', {}),
    ('nonorm_train', "ConfLoss(Regr3D_ShiftInv(L21, norm_mode=''), alpha=0.5)", 'base', {}),
    ('clip', 'Regr3D(L21)', 'base', {'dist_clip': 3.0}),
    ('clip_train', TRAIN, 'base', {'dist_clip': 3.0}),
    ('none', "Regr3D_ScaleShiftInv(L21).with_reduction('none')", 'base', {}),
    ('none_regr3d', "Regr3D(L21, gt_scale=True).with_reduction('none')", 'mixed', {}),
    ('sum', "Regr3D_ShiftInv(L21).with_reduction('sum')", 'base', {}),
    ('compose', '2 * Regr3D(L21) + Regr3D_ScaleShiftInv(L21, gt_scale=True)', 'base', {}),
    ('compose_conf', f'{TRAIN} + 0.5 * {TEST}', 'mixed', {}),
    ('mixed_train', TRAIN, 'mixed', {}),
    ('mixed_test', TEST, 'mixed', {}),
    ('empty_train', TRAIN, 'empty2', {}),
    ('empty_test', TEST, 'empty2', {}),
]


def inputs(name):
    return synth_criterion_batch(**INPUTS[name])


def main():
    sys.path.insert(0, os.environ['DUST3R_REFERENCE'])
    import dust3r.losses as ref
    G, meta = {}, []
    for name in INPUTS:
        for k, view in enumerate(inputs(name)):
            for key, t in view.items():
                G[f'in|{name}|{k}|{key}'] = t.numpy()
    plain_print = builtins.print
    builtins.print = lambda *a, force=False, **kw: plain_print(*a, **kw)
    try:
        for name, expr, src, kw in CASES:
            crit = eval(expr, vars(ref))
            loss, details = crit(*copy.deepcopy(inputs(src)), **kw)
            entry = dict(name=name, expr=expr, inputs=src, kwargs=kw, repr=repr(crit), details=details)
            if isinstance(loss, tuple):   # reduction 'none': ((loss1, mask1), (loss2, mask2))
                for k, (lk, mk) in enumerate(loss):
                    G[f'out|{name}|loss{k + 1}'] = lk.numpy()
                    G[f'out|{name}|mask{k + 1}'] = mk.numpy()
                entry['loss'] = None
            else:
                entry['loss'] = float(loss)
            meta.append(entry)
    finally:
        builtins.print = plain_print
    G['meta'] = np.array(json.dumps(meta))
    np.savez_compressed(os.path.join(HERE, 'criterion.npz'), **G)
    print('wrote', len(meta), 'cases')


if __name__ == '__main__':
    main()
