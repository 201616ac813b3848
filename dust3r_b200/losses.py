"""Evaluation criteria (API mirror of dust3r/losses.py): Regr3D and its shift / scale-invariant variants over L21, ConfLoss, and
the MultiLoss algebra that combines them (`alpha * loss`, `loss_a + loss_b`, `with_reduction('none')`).

Both training recipes of the reference name their criteria as strings evaluated in this module's namespace:
    ConfLoss(Regr3D(L21, norm_mode='avg_dis'), alpha=0.2)        Regr3D_ScaleShiftInv(L21, gt_scale=True)
A criterion is called as `criterion(gt1, gt2, pred1, pred2)` -> (loss, details): gt views carry 'pts3d' (B,H,W,3, world
frame), 'valid_mask' (B,H,W, bool or uint8) and 'camera_pose' (B,4,4); pred1 carries 'pts3d' and 'conf', pred2
'pts3d_in_other_view' and 'conf' (what AsymmetricCroCo3DStereo returns).  The two views may differ in size.

Where the tensors live decides where it runs:
  - all on CUDA: csrc/criterion_ops.cu (d3r_criterion) -- every stage on the device (normalisation sums, the joint medians of
    the shift / scale-invariant variants, the per-pixel distance and confidence weighting, fixed-order fp64 sums), and the
    details fetched with one device->host copy per call;
  - all on the CPU: a torch restatement of the reference (the host port);
  - a mix raises ValueError.
Only norm_mode 'avg_dis' (the one the documented recipes use) or a falsy norm_mode is supported; the reference's other modes
raise NotImplementedError.

Deviations from the reference, all deliberate:
  - the criteria never write into the caller's tensors (with a falsy norm_mode the reference's shift / scale variants shift
    pred['pts3d'] / pred['pts3d_in_other_view'] in place);
  - ConfLoss on a view without any valid pixel prints a warning (the reference's `print(..., force=True)` only works inside its
    training process), counts 0 for that view and reports NaN as its `_pts3d_k` detail;
  - losses are evaluated without autograd: the result carries no graph (evaluation only; training is out of scope);
  - a uint8 valid_mask counts as nonzero = valid.
"""
from __future__ import annotations

import contextlib
from copy import copy, deepcopy

import torch
import torch.nn as nn

from . import _lib
from .inference import get_pred_pts3d
from .utils.geometry import (check_norm_mode, geotrf, get_joint_pointcloud_center_scale, get_joint_pointcloud_depth, inv,
                             normalize_pointcloud)


def Sum(*losses_and_masks):
    """The per-pixel (loss, mask) pairs unchanged when the losses are per pixel, else the sum of the scalar losses."""
    loss, mask = losses_and_masks[0]
    if loss.ndim > 0:
        return losses_and_masks
    for loss2, mask2 in losses_and_masks[1:]:
        loss = loss + loss2
    return loss


class BaseCriterion(nn.Module):
    def __init__(self, reduction='mean'):
        super().__init__()
        self.reduction = reduction


class LLoss(BaseCriterion):
    """L-norm loss between two (..., d) point sets, d in 1..3, reduced by `reduction` ('mean', 'sum' or 'none')."""

    def forward(self, a, b):
        assert a.shape == b.shape and a.ndim >= 2 and 1 <= a.shape[-1] <= 3, f'Bad shape = {a.shape}'
        dist = self.distance(a, b)
        assert dist.ndim == a.ndim - 1
        if self.reduction == 'none':
            return dist
        if self.reduction == 'sum':
            return dist.sum()
        if self.reduction == 'mean':
            return dist.mean() if dist.numel() > 0 else dist.new_zeros(())
        raise ValueError(f'bad {self.reduction=} mode')

    def distance(self, a, b):
        raise NotImplementedError()


class L21Loss(LLoss):
    """Euclidean distance between 3D points."""

    def distance(self, a, b):
        return torch.norm(a - b, dim=-1)


L21 = L21Loss()


class Criterion(nn.Module):
    def __init__(self, criterion=None):
        super().__init__()
        assert isinstance(criterion, BaseCriterion), f'{criterion} is not a proper criterion!'
        self.criterion = copy(criterion)

    def get_name(self):
        return f'{type(self).__name__}({self.criterion})'

    def with_reduction(self, mode='none'):
        res = loss = deepcopy(self)
        while loss is not None:
            assert isinstance(loss, Criterion)
            loss.criterion.reduction = mode
            loss = loss._loss2
        return res


def _as_floats(details):
    """The detail dict with every tensor value replaced by its Python float, all fetched in one copy."""
    keys = [k for k, v in details.items() if torch.is_tensor(v)]
    if keys:
        vals = torch.stack([details[k].detach().reshape(()).float() for k in keys]).tolist()
        details = dict(details)
        details.update(zip(keys, vals))
    return details


class MultiLoss(nn.Module):
    """Combinable losses that keep track of their parts: `loss = MyLoss1() + 0.1 * MyLoss2()`.  Subclasses define get_name()
    and compute_loss(); calling one returns (loss, details)."""

    def __init__(self):
        super().__init__()
        self._alpha = 1
        self._loss2 = None

    def compute_loss(self, *args, **kwargs):
        raise NotImplementedError()

    def get_name(self):
        raise NotImplementedError()

    def __mul__(self, alpha):
        assert isinstance(alpha, (int, float))
        res = copy(self)
        res._alpha = alpha
        return res
    __rmul__ = __mul__

    def __add__(self, loss2):
        assert isinstance(loss2, MultiLoss)
        res = cur = copy(self)
        while cur._loss2 is not None:
            cur = cur._loss2
        cur._loss2 = loss2
        return res

    def __repr__(self):
        name = self.get_name()
        if self._alpha != 1:
            name = f'{self._alpha:g}*{name}'
        if self._loss2:
            name = f'{name} + {self._loss2}'
        return name

    def _chain(self, *args, **kwargs):
        # detail values stay tensors here: forward() converts the whole chain's at once
        loss = self.compute_loss(*args, **kwargs)
        if isinstance(loss, tuple):
            loss, details = loss
        elif loss.ndim == 0:
            details = {self.get_name(): loss}
        else:
            details = {}
        loss = loss * self._alpha
        if self._loss2:
            loss2, details2 = self._loss2._chain(*args, **kwargs)
            loss = loss + loss2
            details |= details2
        return loss, details

    @torch.no_grad()
    def forward(self, *args, **kwargs):
        loss, details = self._chain(*args, **kwargs)
        return loss, _as_floats(details)


# ---------------------------------------------------------------------------------------------------------------------------
# device dispatch

_HOST_PORT = False


@contextlib.contextmanager
def host_port():
    """Within the block, the criteria run the host port's torch code whatever device their tensors are on (this is how
    scripts/criterion_bench.py times the reference's formulation on the GPU)."""
    global _HOST_PORT
    prev, _HOST_PORT = _HOST_PORT, True
    try:
        yield
    finally:
        _HOST_PORT = prev


def _placement(*tensors):
    """'cuda' when every tensor is on one CUDA device, 'cpu' when all are on the CPU; ValueError otherwise."""
    devs = {t.device for t in tensors if torch.is_tensor(t)}
    if _HOST_PORT and len(devs) == 1:
        return 'cpu'
    if all(d.type == 'cpu' for d in devs):
        return 'cpu'
    if all(d.type == 'cuda' for d in devs) and len(devs) == 1:
        return 'cuda'
    raise ValueError(f'criterion inputs must all be on one CUDA device or all on the CPU, got {sorted(map(str, devs))}')


def _pred_pts(pred, second):
    """The predicted points the CUDA path reads: pred1['pts3d'], pred2['pts3d_in_other_view'] (what DUSt3R's heads return)."""
    if 'depth' in pred and 'pseudo_focal' in pred:
        return get_pred_pts3d({}, pred)   # raises
    if second:
        if 'pts3d' in pred:
            raise NotImplementedError('the CUDA criteria read pred2["pts3d_in_other_view"]; a pred2 with "pts3d" and a '
                                      'camera_pose is only supported on CPU tensors')
        return pred['pts3d_in_other_view']
    return get_pred_pts3d({}, pred, use_pose=False)


def _inputs(gt1, gt2, pred1, pred2, conf, strict=False):
    """The tensors a criterion reads; strict: the predicted points as the CUDA path takes them (raises for other layouts)."""
    ts = [gt1['camera_pose'], gt1['pts3d'], gt2['pts3d'], gt1['valid_mask'], gt2['valid_mask']]
    if strict:
        ts += [_pred_pts(pred1, False), _pred_pts(pred2, True)]
    else:
        ts += [v for pred in (pred1, pred2) for k, v in pred.items() if k in ('pts3d', 'pts3d_in_other_view', 'camera_pose')]
    if conf:
        ts += [pred1['conf'], pred2['conf']]
    return ts


_REDUCTIONS = {'mean': 0, 'sum': 1, 'none': 2}
_NORM, _GT_SCALE, _SHIFT, _SCALE, _CONF, _CLIP = 1, 2, 4, 8, 16, 32


def _run_cuda(crit, gt1, gt2, pred1, pred2, dist_clip=None, alpha=None):
    """One d3r_criterion call for a Regr3D-family `crit` (with ConfLoss weighting when alpha is not None).  Returns the fp32
    result vector `out` (see include/dust3r_b200.h) and, with reduction 'none', the per-pixel outputs and their host copy."""
    if not isinstance(crit.criterion, L21Loss) or type(crit.criterion).distance is not L21Loss.distance:
        raise NotImplementedError(f'the CUDA criteria compute the L21 distance, not {crit.criterion}')
    if type(crit) not in (Regr3D, Regr3D_ShiftInv, Regr3D_ScaleInv, Regr3D_ScaleShiftInv):
        raise NotImplementedError(f'{type(crit).__name__} has no CUDA implementation')
    red = crit.criterion.reduction
    if red not in _REDUCTIONS:
        raise ValueError(f'bad {red=} mode')
    ts = _inputs(gt1, gt2, pred1, pred2, alpha is not None, strict=True)
    dev = ts[0].device
    _lib.require_cuda_device(dev)
    pose, g1, g2, m1, m2, p1, p2 = ts[:7]
    B, H1, W1 = g1.shape[:3]
    H2, W2 = g2.shape[1:3]
    assert g1.shape == p1.shape == (B, H1, W1, 3) and g2.shape == p2.shape == (B, H2, W2, 3), 'pointmaps must be (B,H,W,3)'
    assert m1.shape == (B, H1, W1) and m2.shape == (B, H2, W2) and pose.shape == (B, 4, 4), 'bad valid_mask / camera_pose shape'
    f32 = lambda t: t.to(torch.float32).contiguous()
    u8 = lambda m: (m if m.dtype == torch.bool else m != 0).contiguous().view(torch.uint8)
    T = f32(inv(pose))
    g1, g2, p1, p2 = map(f32, (g1, g2, p1, p2))
    m1, m2 = u8(m1), u8(m2)
    c1, c2 = (f32(ts[7]), f32(ts[8])) if alpha is not None else (None, None)
    n1, n2 = H1 * W1, H2 * W2
    flags = (_NORM if crit.norm_mode else 0) | (_GT_SCALE if crit.gt_scale else 0) | (_SHIFT if crit._shift else 0) \
        | (_SCALE if crit._scale else 0) | (_CONF if alpha is not None else 0) | (_CLIP if dist_clip is not None else 0)
    pixels = red == 'none' and alpha is None
    out = torch.empty(8, dtype=torch.float32, device=dev)
    pix = [torch.empty(B * n, dtype=torch.float32, device=dev) for n in (n1, n2)] if pixels else [None, None]
    msk = [torch.empty(s, dtype=torch.bool, device=dev) for s in ((B, H1, W1), (B, H2, W2))] if pixels else [None, None]
    nbytes = int(_lib.get_lib().d3r_criterion_workspace_bytes(B, n1, n2, flags))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    ptr = lambda t: None if t is None else t.data_ptr()
    _lib.launch(dev, 'd3r_criterion', B, n1, n2, flags, _REDUCTIONS[red], float(dist_clip or 0.0), float(alpha or 0.0),
                ptr(T), ptr(g1), ptr(g2), ptr(m1), ptr(m2), ptr(p1), ptr(p2), ptr(c1), ptr(c2), ptr(out),
                ptr(pix[0]), ptr(pix[1]), ptr(msk[0]), ptr(msk[1]), ptr(ws), nbytes)
    return out, pix, msk


def _fetch(out):
    """Host copy of the result vector: (fp32 values as floats, the two valid counts)."""
    h = out.cpu()
    return h[:5].tolist(), h[5:7].view(torch.int32).tolist()


class Regr3D(Criterion, MultiLoss):
    """All 3D points correct, in the frame of view 1's camera (view 1 is the anchor):
        loss1 = |pred_pts1 - inv(pose1) @ gt_pts1|,   loss2 = |pred_pts2_in_view1 - inv(pose1) @ gt_pts2|
    over the valid pixels of each view, after the joint normalisation of each pair (norm_mode; the ground truth keeps its
    scale when gt_scale)."""

    _shift = False
    _scale = False

    def __init__(self, criterion, norm_mode='avg_dis', gt_scale=False):
        super().__init__(criterion)
        check_norm_mode(norm_mode)
        self.norm_mode = norm_mode
        self.gt_scale = gt_scale

    def get_all_pts3d(self, gt1, gt2, pred1, pred2, dist_clip=None):
        in_camera1 = inv(gt1['camera_pose'])
        gt_pts1 = geotrf(in_camera1, gt1['pts3d'])
        gt_pts2 = geotrf(in_camera1, gt2['pts3d'])
        valid1 = gt1['valid_mask'].clone().bool()
        valid2 = gt2['valid_mask'].clone().bool()
        if dist_clip is not None:   # points too far away are invalid
            valid1 = valid1 & (gt_pts1.norm(dim=-1) <= dist_clip)
            valid2 = valid2 & (gt_pts2.norm(dim=-1) <= dist_clip)
        pr_pts1 = get_pred_pts3d(gt1, pred1, use_pose=False)
        pr_pts2 = get_pred_pts3d(gt2, pred2, use_pose=True)
        if self.norm_mode:
            pr_pts1, pr_pts2 = normalize_pointcloud(pr_pts1, pr_pts2, self.norm_mode, valid1, valid2)
        else:   # the variants below shift and scale in place: work on copies of the caller's predictions
            pr_pts1, pr_pts2 = pr_pts1.clone(), pr_pts2.clone()
        if self.norm_mode and not self.gt_scale:
            gt_pts1, gt_pts2 = normalize_pointcloud(gt_pts1, gt_pts2, self.norm_mode, valid1, valid2)
        return gt_pts1, gt_pts2, pr_pts1, pr_pts2, valid1, valid2, {}

    def compute_loss(self, gt1, gt2, pred1, pred2, **kw):
        self_name = type(self).__name__
        if _placement(*_inputs(gt1, gt2, pred1, pred2, False)) == 'cuda':
            if type(self).get_all_pts3d is not Regr3D.get_all_pts3d and kw:   # the variants take no keyword, as the reference
                raise TypeError(f'{self_name}.get_all_pts3d() got an unexpected keyword argument {next(iter(kw))!r}')
            out, pix, msk = _run_cuda(self, gt1, gt2, pred1, pred2, **kw)
            if self.criterion.reduction != 'none':
                return out[4], {self_name + '_pts3d_1': out[0], self_name + '_pts3d_2': out[1]}
            vals, cnt = _fetch(out)
            details = {self_name + '_pts3d_1': vals[0], self_name + '_pts3d_2': vals[1]}
            return ((pix[0][:cnt[0]], msk[0]), (pix[1][:cnt[1]], msk[1])), details
        gt_pts1, gt_pts2, pred_pts1, pred_pts2, mask1, mask2, monitoring = self.get_all_pts3d(gt1, gt2, pred1, pred2, **kw)
        l1 = self.criterion(pred_pts1[mask1], gt_pts1[mask1])
        l2 = self.criterion(pred_pts2[mask2], gt_pts2[mask2])
        details = {self_name + '_pts3d_1': l1.mean(), self_name + '_pts3d_2': l2.mean()}
        return Sum((l1, mask1), (l2, mask2)), (details | monitoring)


class ConfLoss(MultiLoss):
    """A per-pixel regression loss weighted by the predicted confidence: conf * loss - alpha * log(conf), averaged over the
    valid pixels of each view (high confidence conf = 10: 10 * loss - alpha * log(10); low conf = 0.1: loss / 10 + ...)."""

    def __init__(self, pixel_loss, alpha=1):
        super().__init__()
        assert alpha > 0
        self.alpha = alpha
        self.pixel_loss = pixel_loss.with_reduction('none')

    def get_name(self):
        return f'ConfLoss({self.pixel_loss})'

    def get_conf_log(self, x):
        return x, torch.log(x)

    def compute_loss(self, gt1, gt2, pred1, pred2, **kw):
        if _placement(*_inputs(gt1, gt2, pred1, pred2, True)) == 'cuda':
            return self._compute_loss_cuda(gt1, gt2, pred1, pred2, **kw)
        ((loss1, msk1), (loss2, msk2)), details = self.pixel_loss(gt1, gt2, pred1, pred2, **kw)
        for k, loss in enumerate((loss1, loss2)):
            if loss.numel() == 0:
                print(f'NO VALID POINTS in img{k + 1}')
        conf1, log_conf1 = self.get_conf_log(pred1['conf'][msk1])
        conf2, log_conf2 = self.get_conf_log(pred2['conf'][msk2])
        conf_loss1 = loss1 * conf1 - self.alpha * log_conf1
        conf_loss2 = loss2 * conf2 - self.alpha * log_conf2
        # average; a view without valid pixels counts 0
        conf_loss1 = conf_loss1.mean() if conf_loss1.numel() > 0 else conf_loss1.new_zeros(())
        conf_loss2 = conf_loss2.mean() if conf_loss2.numel() > 0 else conf_loss2.new_zeros(())
        return conf_loss1 + conf_loss2, dict(conf_loss_1=conf_loss1, conf_loss2=conf_loss2, **details)

    def _compute_loss_cuda(self, gt1, gt2, pred1, pred2, **kw):
        pl = self.pixel_loss
        if not isinstance(pl, Regr3D) or pl._loss2 is not None or pl._alpha != 1 or type(self).get_conf_log is not ConfLoss.get_conf_log:
            raise NotImplementedError(f'{self.get_name()} has no CUDA implementation: the CUDA ConfLoss weights one Regr3D-family '
                                      'criterion with conf * loss - alpha * log(conf)')
        if type(pl).get_all_pts3d is not Regr3D.get_all_pts3d and kw:
            raise TypeError(f'{type(pl).__name__}.get_all_pts3d() got an unexpected keyword argument {next(iter(kw))!r}')
        out, _, _ = _run_cuda(pl, gt1, gt2, pred1, pred2, alpha=self.alpha, **kw)
        vals, cnt = _fetch(out)
        for k in range(2):
            if cnt[k] == 0:
                print(f'NO VALID POINTS in img{k + 1}')
        name = type(pl).__name__
        return out[4], dict(conf_loss_1=vals[2], conf_loss2=vals[3], **{name + '_pts3d_1': vals[0], name + '_pts3d_2': vals[1]})


class Regr3D_ShiftInv(Regr3D):
    """Regr3D invariant to a depth shift: gt and prediction each lose the median depth of their valid points (both views)."""

    _shift = True

    def get_all_pts3d(self, gt1, gt2, pred1, pred2):
        gt_pts1, gt_pts2, pred_pts1, pred_pts2, mask1, mask2, monitoring = super().get_all_pts3d(gt1, gt2, pred1, pred2)
        gt_z1, gt_z2 = gt_pts1[..., 2], gt_pts2[..., 2]
        pred_z1, pred_z2 = pred_pts1[..., 2], pred_pts2[..., 2]
        gt_shift_z = get_joint_pointcloud_depth(gt_z1, gt_z2, mask1, mask2)[:, None, None]
        pred_shift_z = get_joint_pointcloud_depth(pred_z1, pred_z2, mask1, mask2)[:, None, None]
        gt_z1 -= gt_shift_z
        gt_z2 -= gt_shift_z
        pred_z1 -= pred_shift_z
        pred_z2 -= pred_shift_z
        return gt_pts1, gt_pts2, pred_pts1, pred_pts2, mask1, mask2, monitoring


class Regr3D_ScaleInv(Regr3D):
    """Regr3D invariant to scale: gt and prediction are each divided by the median distance of their valid points to their
    per-coordinate median (the prediction's clipped to [1e-3, 1e3]); with gt_scale the prediction is brought to the gt's scale."""

    _scale = True

    def get_all_pts3d(self, gt1, gt2, pred1, pred2):
        gt_pts1, gt_pts2, pred_pts1, pred_pts2, mask1, mask2, monitoring = super().get_all_pts3d(gt1, gt2, pred1, pred2)
        _, gt_scale = get_joint_pointcloud_center_scale(gt_pts1, gt_pts2, mask1, mask2)
        _, pred_scale = get_joint_pointcloud_center_scale(pred_pts1, pred_pts2, mask1, mask2)
        pred_scale = pred_scale.clip(min=1e-3, max=1e3)
        if self.gt_scale:
            pred_pts1 *= gt_scale / pred_scale
            pred_pts2 *= gt_scale / pred_scale
        else:
            gt_pts1 /= gt_scale
            gt_pts2 /= gt_scale
            pred_pts1 /= pred_scale
            pred_pts2 /= pred_scale
        return gt_pts1, gt_pts2, pred_pts1, pred_pts2, mask1, mask2, monitoring


class Regr3D_ScaleShiftInv(Regr3D_ScaleInv, Regr3D_ShiftInv):
    """Shift, then scale invariance (the MRO runs Regr3D_ShiftInv's step before Regr3D_ScaleInv's)."""


@torch.no_grad()
def cuda_nanmedian(x):
    """torch.nanmedian(x, dim=-1).values for a CUDA tensor, by the segmented radix select every median of the criteria uses
    (d3r_segmented_nanmedian): the lower median of the non-NaN values of each row, NaN for a row without one, in fp32."""
    if not x.is_cuda:
        raise ValueError('cuda_nanmedian takes a CUDA tensor')
    dev = _lib.require_cuda_device(x.device)
    rows = x.reshape(-1, x.shape[-1]).to(torch.float32).contiguous()
    out = torch.empty(rows.shape[0], dtype=torch.float32, device=dev)
    nbytes = int(_lib.get_lib().d3r_nanmedian_workspace_bytes(rows.shape[0]))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _lib.launch(dev, 'd3r_segmented_nanmedian', rows.shape[0], rows.shape[1], rows.data_ptr(), out.data_ptr(), ws.data_ptr(), nbytes)
    return out.reshape(x.shape[:-1])
