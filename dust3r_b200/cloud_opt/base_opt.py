"""Scene container + alignment loop driver (API mirror of dust3r/cloud_opt/base_opt.py).

The reference runs `niter` x (python forward over torch ops + autograd + torch.optim.Adam + a
float(loss) sync).  Here `compute_global_alignment` hands the whole loop to the fused CUDA step
(csrc/align_step.cu) through AlignEngine; this module only keeps the reference's object model
(edges, pred_i/pred_j/conf_i/conf_j dictionaries keyed "i_j", im_conf, pw_poses, pw_adaptors,
state_dict split, getters) so callers written against the reference keep working.
"""
from __future__ import annotations

from copy import deepcopy

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from ..utils.geometry import inv
from ..utils.image import rgb
from ..viz import segment_sky
from . import pose_param
from .commons import ALL_DISTS, NoGradParamDict, edge_str, get_conf_trf, get_imshapes
from .engine import AlignEngine
from .pointcloud_filter import clean_pointcloud
from .scene_ops import segment_sky_host_images


class BasePCOptimizer(nn.Module):
    """Graph node = image, graph edge = one pairwise prediction (pred1, pred2).
    Constructor arguments follow base_opt.py:44-53."""

    # attributes shared (not copied) when one optimizer is built from another one
    _SCENE_ATTRS = ('edges', 'is_symmetrized', 'dist', 'n_imgs', 'pred_i', 'pred_j', 'imshapes', 'min_conf_thr', 'conf_thr',
                    'conf_i', 'conf_j', 'im_conf', 'base_scale', 'norm_pw_scale', 'POSE_DIM', 'pw_poses', 'pw_adaptors',
                    'has_im_poses', 'rand_pose', 'imgs', 'verbose', 'conf_mode', 'conf_trf', 'pw_break', 'align_kernel')

    def __init__(self, *args, **kwargs):
        if len(args) == 1 and not kwargs:
            # BasePCOptimizer(other): take over a deep copy of the other optimizer's scene (base_opt.py:45-53)
            source = deepcopy(args[0])
            for name in self._SCENE_ATTRS:
                self.__dict__[name] = source[name]
        else:
            self._init_from_views(*args, **kwargs)

    def _init_from_views(self, view1, view2, pred1, pred2,
                         dist='l1', conf='log', min_conf_thr=3, base_scale=0.5,
                         allow_pw_adaptors=False, pw_break=20, rand_pose=torch.randn,
                         iterationsCount=None, verbose=True, kernel='auto', imshapes=None):
        """Scene graph from the output of inference(): view*['idx'] give the image ids of every pair, pred1 / pred2 the
        two pointmaps (+ confidences) of every pair, both expressed in the first image's camera frame.

        imshapes (extension): (H, W) of every image, for the rows of inference_sharded(keep='owned'), where pred1 / pred2
        hold None for the pairs (or view-2 halves) this rank does not keep.  The per-edge dictionaries then hold only the
        kept entries, and im_conf only this rank's maxima until distributed.global_aligner_sharded shares it."""
        super().__init__()
        if dist not in ALL_DISTS:
            raise KeyError(dist)
        self.dist, self.verbose = dist, verbose
        self.align_kernel = kernel       # extension: 'auto' | 'stream' | 'general' (which fused CUDA step runs the loop)

        # ---- graph
        for view in (view1, view2):
            if not isinstance(view['idx'], list):
                view['idx'] = view['idx'].tolist()
        first, second = view1['idx'], view2['idx']
        self.edges = [(int(i), int(j)) for i, j in zip(first, second)]
        self.is_symmetrized = {(j, i) for i, j in self.edges} == set(self.edges)
        self.n_imgs = self._check_edges()

        # ---- observations, one entry per directed pair "i_j"
        def per_edge(stacked):
            return NoGradParamDict({key: stacked[e] for e, key in enumerate(self.str_edges) if stacked[e] is not None})
        pts_i, pts_j = pred1['pts3d'], pred2['pts3d_in_other_view']
        # equal-size scenes arrive as 4 stacked tensors: remember them so that .to(device) moves 4 buffers (one H2D
        # copy each, or none at all when inference(keep_on_device=True) / the all-gather left them in HBM) and the
        # per-edge dictionaries stay views of them, instead of 4E separate parameter copies
        stacks = (pts_i, pts_j, pred1['conf'], pred2['conf'])
        self._obs_stacks = stacks if all(torch.is_tensor(t) for t in stacks) else None
        self.pred_i, self.pred_j = per_edge(pts_i), per_edge(pts_j)
        self.imshapes = [tuple(hw) for hw in imshapes] if imshapes is not None else get_imshapes(self.edges, pts_i, pts_j)
        self.min_conf_thr = min_conf_thr
        self.conf_mode, self.conf_trf = conf, get_conf_trf(conf)
        self.conf_i, self.conf_j = per_edge(pred1['conf']), per_edge(pred2['conf'])
        self.im_conf = self._compute_img_conf(pred1['conf'], pred2['conf'])
        self.im_conf.requires_grad_(False)

        # ---- pairwise similarity transforms (pose + log-scale) and optional anisotropic adaptors
        self.base_scale, self.norm_pw_scale, self.pw_break = base_scale, True, pw_break
        self.POSE_DIM = 7
        self.rand_pose = rand_pose
        self.pw_poses = nn.Parameter(rand_pose((self.n_edges, 1 + self.POSE_DIM)))
        self.pw_adaptors = nn.Parameter(torch.zeros((self.n_edges, 2)), requires_grad=bool(allow_pw_adaptors))
        self.has_im_poses = False

        # ---- colours for visualisation / export
        self.imgs = None
        if 'img' in view1 and 'img' in view2:
            canvas = [torch.zeros((3,) + tuple(hw)) for hw in self.imshapes]
            for e, (i, j) in enumerate(zip(first, second)):
                canvas[i], canvas[j] = view1['img'][e], view2['img'][e]
            self.imgs = rgb(canvas)
        self._engine = None

    # ---------------------------------------------------------------- bookkeeping
    @property
    def n_edges(self):
        return len(self.edges)

    @property
    def str_edges(self):
        return [edge_str(i, j) for i, j in self.edges]

    @property
    def imsizes(self):
        return [(w, h) for h, w in self.imshapes]

    @property
    def device(self):
        return next(iter(self.parameters())).device

    def state_dict(self, trainable=True):
        every = super().state_dict()
        observed = ('_', 'pred_i.', 'pred_j.', 'conf_i.', 'conf_j.')
        return {k: v for k, v in every.items() if k.startswith(observed) != trainable}

    def load_state_dict(self, data):
        self._engine = None
        return super().load_state_dict(self.state_dict(trainable=False) | data)

    _OBS_DICTS = ('pred_i', 'pred_j', 'conf_i', 'conf_j')

    def _apply(self, fn, *a, **kw):
        self._engine = None  # device / dtype moves invalidate the packed observation buffer
        stacks = self.__dict__.get('_obs_stacks')
        if stacks is None:
            return super()._apply(fn, *a, **kw)
        # move the 4 stacked observation tensors once and re-create the per-edge views on the result
        held = {name: self._modules.pop(name) for name in self._OBS_DICTS}
        try:
            super()._apply(fn, *a, **kw)
            moved = tuple(fn(t) for t in stacks)
        except Exception:
            self._modules.update(held)
            raise
        self._obs_stacks = moved
        keys = self.str_edges
        for name, stacked in zip(self._OBS_DICTS, moved):
            self._modules[name] = NoGradParamDict({key: stacked[e] for e, key in enumerate(keys)})
        return self

    def _check_edges(self):
        indices = sorted({i for edge in self.edges for i in edge})
        assert indices == list(range(len(indices))), 'bad pair indices: missing values '
        return len(indices)

    @torch.no_grad()
    def _compute_img_conf(self, pred1_conf, pred2_conf):
        """Per-image maximum of the confidences of its entries (entries this rank does not keep are None and skipped)."""
        first = next((c for confs in (pred1_conf, pred2_conf) for c in confs if c is not None), None)
        dev = first.device if first is not None else None
        im_conf = nn.ParameterList([torch.zeros(hw, device=dev) for hw in self.imshapes])
        for e, (i, j) in enumerate(self.edges):
            if pred1_conf[e] is not None:
                im_conf[i] = torch.maximum(im_conf[i], pred1_conf[e])
            if pred2_conf[e] is not None:
                im_conf[j] = torch.maximum(im_conf[j], pred2_conf[e])
        return im_conf

    # ---------------------------------------------------------------- pairwise poses
    def get_adaptors(self):
        adapt = self.pw_adaptors
        adapt = torch.cat((adapt[:, 0:1], adapt), dim=-1)
        if self.norm_pw_scale:
            adapt = adapt - adapt.mean(dim=1, keepdim=True)
        return (adapt / self.pw_break).exp()

    def _get_poses(self, poses):
        return pose_param.rows_to_matrices(poses)

    def _set_pose(self, poses, idx, R, T=None, scale=None, force=False):
        """Write a rotation / translation (or a 4x4 passed as R) and optionally a scale into pose row `idx`; frozen
        rows are left alone unless `force`.  Returns the row's parameter."""
        target = poses[idx]
        if not (force or target.requires_grad):
            return target
        if R is not None and tuple(R.shape) == (4, 4):
            assert T is None
            R, T = pose_param.split_rigid(R)
        if scale is not None:
            assert poses.shape[-1] in (8, 13)
        pose_param.write_row(target.data, R, T, scale)
        return target

    def get_pw_norm_scale_factor(self):
        return pose_param.scale_gauge(self.pw_poses[:, -1], self.base_scale, self.norm_pw_scale)

    def get_pw_scale(self):
        return self.pw_poses[:, -1].exp() * self.get_pw_norm_scale_factor()

    def get_pw_poses(self):
        """(E,4,4) similarity transforms: the rigid part of every pairwise pose with its first three rows scaled."""
        out = self._get_poses(self.pw_poses).clone()
        out[:, :3] *= self.get_pw_scale().view(-1, 1, 1)
        return out

    # ---------------------------------------------------------------- accessors
    def get_masks(self):
        return [(conf > self.min_conf_thr) for conf in self.im_conf]

    def get_conf(self, mode=None):
        trf = self.conf_trf if mode is None else get_conf_trf(mode)
        return [trf(c) for c in self.im_conf]

    def depth_to_pts3d(self):
        raise NotImplementedError()

    def get_pts3d(self, raw=False):
        res = self.depth_to_pts3d()
        if not raw:
            res = [dm[:h * w].view(h, w, 3) for dm, (h, w) in zip(res, self.imshapes)]
        return res

    def _set_focal(self, idx, focal, force=False):
        raise NotImplementedError()

    def get_focals(self):
        raise NotImplementedError()

    def get_known_focal_mask(self):
        raise NotImplementedError()

    def get_principal_points(self):
        raise NotImplementedError()

    def get_im_poses(self):
        raise NotImplementedError()

    def _set_depthmap(self, idx, depth, force=False):
        raise NotImplementedError()

    def get_depthmaps(self, raw=False):
        raise NotImplementedError()

    def clean_pointcloud(self, **kw):
        cams = inv(self.get_im_poses())
        K = self.get_intrinsics()
        depthmaps = self.get_depthmaps()
        all_pts3d = self.get_pts3d()
        new_im_confs = clean_pointcloud(self.im_conf, K, cams, depthmaps, all_pts3d, **kw)
        for i, new_conf in enumerate(new_im_confs):
            self.im_conf[i].data[:] = new_conf
        return self

    # ---------------------------------------------------------------- engine plumbing
    def _engine_variant(self):
        return 'per_edge'   # BasePCOptimizer.forward (base_opt.py:246-273): per-edge means / n_edges

    def _engine_pix_stride(self):
        return None

    def _build_engine(self):
        """The scene's AlignEngine; a scene from distributed.global_aligner_sharded gets the engine of this rank's images."""
        dev = self.device
        keys = self.str_edges
        shard = self.__dict__.get('_align_shard')
        # a scene of kept rows (inference_sharded(keep='owned')) lacks the entries of other ranks' images: the engine
        # packs only its own images' entries and never reads those
        self._engine = AlignEngine(
            self.edges, self.imshapes,
            *([obs.get(k) for k in keys] for obs in (self.pred_i, self.pred_j, self.conf_i, self.conf_j)),
            device=dev, conf_mode=self.conf_mode, dist=self.dist, variant=self._engine_variant(), pix_stride=self._engine_pix_stride(),
            base_scale=self.base_scale, pw_break=self.pw_break,
            focal_break=getattr(self, 'focal_break', getattr(self, 'focal_brake', 20)),
            kernel=getattr(self, 'align_kernel', 'auto'),
            shards=shard.shards if shard is not None else None, group=shard.group if shard is not None else None)
        return self._engine

    def _engine_push(self, eng):
        """copy python-side parameters into the engine buffers; returns a finaliser that copies back"""
        raise NotImplementedError()

    def _get_engine(self):
        eng = self._engine if self._engine is not None else self._build_engine()
        return eng

    def _engine_params(self):
        """Every parameter the engine optimises, in the order of _engine_grads."""
        raise NotImplementedError()

    def _engine_grads(self, eng, logd_grad, small_grad):
        """Gradients of _engine_params() from the flat gradients of AlignEngine.loss_and_grad (or sharded_loss_and_grad),
        each shaped like its parameter."""
        raise NotImplementedError()

    def forward(self, ret_details=False):
        """Objective at the current parameters (a CUDA scalar tensor).  With grad mode on and a parameter that requires
        grad, the loss carries an autograd graph: backward() hands the fused kernel's analytic gradients to the
        parameters.  ret_details=True also returns the (n, n) CPU tensor of per-edge losses li + lj (-1 off the edges).
        On a scene of distributed.global_aligner_sharded this is a collective, like compute_global_alignment: every rank of
        the group calls it, the objective is taken at rank 0's parameters, and every rank gets the same loss, details and
        .grad (backward() itself runs no collective)."""
        eng = self._get_engine()
        self._engine_push(eng)
        params = self._engine_params()
        if not ret_details and not (torch.is_grad_enabled() and any(p.requires_grad for p in params)):
            return eng.evaluate_loss()
        loss_and_grad = eng.sharded_loss_and_grad if eng.shards is not None else eng.loss_and_grad
        loss, logd_grad, small_grad, ent = loss_and_grad(entry_loss=ret_details)
        loss = _FusedObjective.apply(loss, self._engine_grads(eng, logd_grad, small_grad), *params)
        if not ret_details:
            return loss
        # per-edge pixel means: the entries carry the coefficient 1 / (area * n_edges)
        per_edge = (ent.sum(dim=1) * self.n_edges).cpu()
        details = -torch.ones((self.n_imgs, self.n_imgs))
        for e, (i, j) in enumerate(self.edges):
            details[i, j] = per_edge[e]
        return loss, details

    @torch.no_grad()
    def compute_global_alignment(self, init=None, niter_PnP=10, **kw):
        if init is None:
            pass
        elif init in ('msp', 'mst'):
            from . import init_im_poses as init_fun
            init_fun.init_minimum_spanning_tree(self, niter_PnP=niter_PnP)
        elif init == 'known_poses':
            from . import init_im_poses as init_fun
            init_fun.init_from_known_poses(self, min_conf_thr=self.min_conf_thr, niter_PnP=niter_PnP)
        else:
            raise ValueError(f'bad value for {init=}')
        return global_alignment_loop(self, **kw)

    @torch.no_grad()
    def mask_sky(self):
        """base_opt.py:289-295: a copy of the scene whose im_conf is 0 on the sky pixels of every image (viz.segment_sky); the
        scene itself is left as it is.  On a CUDA scene one batched kernel call segments all images.  The copy does not share
        the alignment engine: it builds its own when it is next aligned."""
        if self.imgs is None:
            raise ValueError('mask_sky needs the images: build the scene from views that carry "img"')
        res = deepcopy(self, {id(self.__dict__.get('_engine')): None})    # the memo entry copies the engine as None
        res._engine = None
        if self.device.type == 'cuda':
            skies = segment_sky_host_images(self.imgs, self.device)
        else:
            skies = [segment_sky(img) for img in self.imgs]
        for conf, sky in zip(res.im_conf, skies):
            conf[sky.to(conf.device)] = 0
        return res

    def show(self, *a, **kw):
        raise NotImplementedError('visualisation is outside the two hot paths (SURVEY §2 #14)')


class _FusedObjective(torch.autograd.Function):
    """Attaches the gradients the fused kernel computed with the loss to the parameters: backward returns
    grad_output x the stored gradient of every parameter that requires grad."""

    @staticmethod
    def forward(ctx, loss, grads, *params):
        ctx.grads = grads
        return loss.clone()

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        need = ctx.needs_input_grad[2:]
        return (None, None) + tuple(g * grad_output if want else None for g, want in zip(ctx.grads, need))


@torch.no_grad()
def global_alignment_loop(net, lr=0.01, niter=300, schedule='cosine', lr_min=1e-6):
    """base_opt.py:326-349.  Returns float(loss of the last iteration)."""
    if not any(p.requires_grad for p in net.parameters()):
        return net
    if net.verbose:
        print('Global alignement - optimizing for:')
        print([name for name, value in net.named_parameters() if value.requires_grad])
    if schedule not in ('cosine', 'linear'):
        raise ValueError(f'bad lr {schedule=}')
    eng = net._get_engine()
    pull = net._engine_push(eng)
    losses = eng.run(niter, lr=lr, schedule=schedule, lr_min=lr_min)
    pull()
    net.last_losses = losses
    if niter <= 0:
        return float('inf')
    loss = float(losses[-1])  # the only host sync of the loop
    eng.check_overflow()
    if net.verbose:
        print(f' final loss={loss:g} after {niter} iterations')
    return loss
