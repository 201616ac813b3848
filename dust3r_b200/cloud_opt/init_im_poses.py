"""Initialisation of the global aligner before the fused loop runs (`init='mst'` / `'known_poses'`; SURVEY §8f rank 1;
reference behaviour: dust3r/cloud_opt/init_im_poses.py:23-316).

'mst': the pair graph is weighted by pair confidence; along its maximum-confidence spanning tree, starting from the
best pair, every new image is attached to the growing world point cloud by a weighted similarity registration
(Umeyama) of the pair's prediction of an already placed image onto that image's world points.  Focals come from each
image's own pointmap (Weiszfeld IRLS), camera poses from the registrations or, failing that, PnP-RANSAC (cv2); finally
every pairwise pose is registered onto the world cloud and depths are read off in each camera.  The heavy reductions
are torch ops on the optimizer's device (GPU when the scene lives there); scipy / cv2 parts run on the host.
`roma.rigid_points_registration` of the reference is replaced by commons.rigid_points_registration."""
from __future__ import annotations

from collections import deque
from functools import cache

import numpy as np
import scipy.sparse as sp
import torch

from ..post_process import estimate_focal_knowing_depth
from ..utils.device import to_numpy
from ..utils.geometry import geotrf, inv
from . import commons, owned
from .commons import compute_edge_scores, edge_str, i_j_ij


# ---------------------------------------------------------------------------------------------- small geometry helpers
def sRT_to_4x4(scale, R, T, device):
    """Similarity x -> scale * R x + T as a 4x4 matrix."""
    mat = torch.eye(4, device=device)
    mat[:3, :3] = scale * torch.as_tensor(R, dtype=torch.float32, device=device)
    mat[:3, 3] = torch.as_tensor(T, dtype=torch.float32, device=device).reshape(3)
    return mat


def rigid_points_registration(pts1, pts2, conf):
    """Weighted Umeyama: (scale, R, T) with pts2 ~ scale * R pts1 + T, weights = conf."""
    R, T, scale = commons.rigid_points_registration(pts1.reshape(-1, 3), pts2.reshape(-1, 3), weights=conf.reshape(-1),
                                                    compute_scaling=True)
    return scale, R, T


def estimate_focal(pts3d_i, pp=None):
    """Focal (pixels) of the camera that produced pointmap pts3d_i (H,W,3), principal point at the centre by default."""
    H, W, C = pts3d_i.shape
    assert C == 3
    if pp is None:
        pp = torch.tensor((W / 2, H / 2), device=pts3d_i.device)
    return float(estimate_focal_knowing_depth(pts3d_i[None], pp[None], focal_mode='weiszfeld').reshape(-1)[0])


@cache
def pixel_grid(H, W):
    """(H, W, 2) float32 array of (x, y) pixel coordinates."""
    return np.stack(np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32)), axis=-1)


def fast_pnp(pts3d, focal, msk, device, pp=None, niter_PnP=10):
    """RANSAC-PnP of a pointmap against its own pixel grid -> (focal, cam2world), or None when fewer than 4 points
    are usable / no hypothesis succeeds.  With focal=None, 21 log-spaced candidates are tried and the one with most
    inliers wins."""
    import cv2
    if msk.sum() < 4:
        return None
    pts3d, msk = to_numpy(pts3d), to_numpy(msk)
    H, W, C = pts3d.shape
    assert C == 3
    px = pixel_grid(H, W)
    candidates = [focal] if focal is not None else np.geomspace(max(W, H) / 2, max(W, H) * 3, 21)
    cx, cy = (W / 2, H / 2) if pp is None else to_numpy(pp)
    winner = None          # (inlier count, rvec, tvec, focal)
    for f in candidates:
        K = np.float32([(f, 0, cx), (0, f, cy), (0, 0, 1)])
        ok, rvec, tvec, inliers = cv2.solvePnPRansac(pts3d[msk], px[msk], K, None, iterationsCount=niter_PnP, reprojectionError=5,
                                                     flags=cv2.SOLVEPNP_SQPNP)
        if ok and (winner is None or len(inliers) > winner[0]):
            winner = (len(inliers), rvec, tvec, f)
    if winner is None or winner[0] == 0:
        return None
    _, rvec, tvec, f = winner
    world2cam = sRT_to_4x4(1, torch.from_numpy(cv2.Rodrigues(rvec)[0]).float(), torch.from_numpy(tvec).float(), device)
    return f, inv(world2cam)


def get_known_poses(self):
    """(count, mask, poses) of the frozen image poses of an optimizer; (0, None, None) without image poses."""
    if not self.has_im_poses:
        return 0, None, None
    frozen = torch.tensor([not prm.requires_grad for prm in self.im_poses])
    return frozen.sum(), frozen, self.get_im_poses()


def get_known_focals(self):
    if not self.has_im_poses:
        return 0, None, None
    frozen = self.get_known_focal_mask()
    return frozen.sum(), frozen, self.get_focals()


def align_multiple_poses(src_poses, target_poses):
    """Similarity (s, R, T) taking the cameras `src_poses` onto `target_poses` (both (N,4,4) cam2world): registers the
    camera centres plus one point a little way along every optical axis, so orientation counts as well."""
    assert src_poses.shape == target_poses.shape and tuple(src_poses.shape[1:]) == (4, 4)

    def anchors(poses):
        centres = poses[:, :3, 3]
        gaps = torch.cdist(centres, centres)
        upper = torch.triu_indices(len(centres), len(centres), offset=1)
        step = float(gaps[upper[0], upper[1]].median()) / 100
        return torch.cat((centres, centres + step * poses[:, :3, 2]))
    R, T, s = commons.rigid_points_registration(anchors(src_poses), anchors(target_poses), compute_scaling=True)
    return s, R, T


def dict_to_sparse_graph(dic):
    """{(i, j): weight} -> scipy sparse matrix."""
    size = 1 + max(max(edge) for edge in dic)
    graph = sp.dok_array((size, size))
    for edge, weight in dic.items():
        graph[edge] = weight
    return graph


# ------------------------------------------------------------------------------------------------ spanning-tree growth
def minimum_spanning_tree(imshapes, edges, pred_i, pred_j, conf_i, conf_j, im_conf, min_conf_thr, device,
                          has_im_poses=True, niter_PnP=10, verbose=True, scores=None):
    """Returns (world pointmap per image, tree edges in attachment order, focals, cam2world poses).  scores: the
    {(i, j): score} of compute_edge_scores when already known."""
    n_imgs = len(imshapes)
    if scores is None:
        scores = compute_edge_scores(map(i_j_ij, edges), conf_i, conf_j)
    # scipy computes MINIMUM spanning trees: negate the confidences
    graph = -dict_to_sparse_graph(scores)
    tree = sp.csgraph.minimum_spanning_tree(graph).tocoo()
    # best edge on the right; an edge that cannot be attached yet goes back to the left end (lowest priority)
    queue = deque(sorted(zip(-tree.data, tree.row, tree.col)))
    world = [None] * n_imgs
    poses = [None] * n_imgs
    focals = [None] * n_imgs
    placed = set()
    attached = []

    def say(i, j, score, star_i, star_j):
        if verbose:
            print(f' init edge ({i}{"*" * star_i},{j}{"*" * star_j}) {score=}')

    # the strongest pair fixes the world frame: its first image is the origin
    score, i, j = queue.pop()
    say(i, j, score, True, True)
    key = edge_str(i, j)
    world[i], world[j] = pred_i[key].clone(), pred_j[key].clone()
    placed.update((i, j))
    attached.append((i, j))
    if has_im_poses:
        poses[i] = torch.eye(4, device=device)
        focals[i] = estimate_focal(pred_i[key])

    while queue:
        score, i, j = queue.pop()
        if focals[i] is None:
            # NB: the reference evaluates this with the key of the PREVIOUSLY processed edge (init_im_poses.py:154-155);
            # reproduced so that initial focals agree
            focals[i] = estimate_focal(pred_i[key])
        if i in placed:           # (i, j): i known, attach j through the pair's view of i
            assert j not in placed
            say(i, j, score, False, True)
            key = edge_str(i, j)
            s, R, T = rigid_points_registration(pred_i[key], world[i], conf=conf_i[key])
            world[j] = geotrf(sRT_to_4x4(s, R, T, device), pred_j[key])
            placed.add(j)
        elif j in placed:         # (i, j): j known, attach i through the pair's view of j
            assert i not in placed
            say(i, j, score, True, False)
            key = edge_str(i, j)
            s, R, T = rigid_points_registration(pred_j[key], world[j], conf=conf_j[key])
            world[i] = geotrf(sRT_to_4x4(s, R, T, device), pred_i[key])
            placed.add(i)
        else:                     # neither end placed yet: retry after everything else
            queue.appendleft((score, i, j))
            continue
        attached.append((i, j))
        if has_im_poses and poses[i] is None:
            # camera i is the reference camera of this pair: the registration (without scale) is its pose
            poses[i] = sRT_to_4x4(1, R, T, device)

    if not has_im_poses:
        return world, attached, None, None

    # images that never were the first image of a processed pair: focal from their best pair, pose by PnP
    # most confident (most negative weight) first
    by_score = np.array(list(graph.keys()))[np.argsort(list(graph.values()))].tolist()
    for i, j in by_score:
        if focals[i] is None:
            focals[i] = estimate_focal(pred_i[edge_str(i, j)])
    for i in range(n_imgs):
        if poses[i] is None:
            solved = fast_pnp(world[i], focals[i], msk=im_conf[i] > min_conf_thr, device=device, niter_PnP=niter_PnP)
            if solved:
                focals[i], poses[i] = solved
        if poses[i] is None:
            poses[i] = torch.eye(4, device=device)
    return world, attached, focals, torch.stack(poses)


def init_from_pts3d(self, pts3d, im_focals, im_poses):
    """Write a world point cloud (+ focals, poses) into an optimizer's parameters."""
    n_known, known_msk, known_poses = get_known_poses(self)
    if n_known == 1:
        raise NotImplementedError("Would be simpler to just align everything afterwards on the single known pose")
    if n_known > 1:
        # move the whole initial scene onto the frozen cameras
        s, R, T = align_multiple_poses(im_poses[known_msk], known_poses[known_msk])
        to_known = sRT_to_4x4(s, R, T, device=known_poses.device)
        im_poses = to_known @ im_poses
        im_poses[:, :3, :3] /= s
        for cloud in pts3d:
            cloud[:] = geotrf(to_known, cloud)

    # pairwise similarity of every pair onto the world cloud; a scene of kept rows registers the edges whose row it keeps
    # and takes the others' from their keepers
    partial = owned.shard_of(self) is not None
    mine = owned.keeps_edge(self) if partial else None
    for e, (i, j) in enumerate(self.edges):
        if partial and not mine[e]:
            continue
        key = edge_str(i, j)
        s, R, T = rigid_points_registration(self.pred_i[key], pts3d[i], conf=self.conf_i[key])
        self._set_pose(self.pw_poses, e, R, T, scale=s)
    if partial and self.pw_poses.requires_grad:
        owned.share_edge_rows(self, self.pw_poses)

    # fix the scale gauge the way the objective does
    gauge = self.get_pw_norm_scale_factor()
    im_poses[:, :3, 3] *= gauge
    for cloud in pts3d:
        cloud *= gauge

    if self.has_im_poses:
        for i in range(self.n_imgs):
            cam2world = im_poses[i]
            self._set_depthmap(i, geotrf(inv(cam2world), pts3d[i])[..., 2])
            self._set_pose(self.im_poses, i, cam2world)
            if im_focals[i] is not None:
                self._set_focal(i, im_focals[i])
    if self.verbose:
        print(' init loss =', float(self()))


@torch.no_grad()
def init_minimum_spanning_tree(self, **kw):
    rows, scores = (self.pred_i, self.pred_j, self.conf_i, self.conf_j), None
    if owned.shard_of(self) is not None:     # kept rows: scores from their keepers, the rows the walk reads broadcast
        rows, scores = owned.kept_rows(self), owned.edge_scores(self)
    pts3d, _, im_focals, im_poses = minimum_spanning_tree(self.imshapes, self.edges, *rows, self.im_conf, self.min_conf_thr,
                                                          self.device, has_im_poses=self.has_im_poses, verbose=self.verbose,
                                                          scores=scores, **kw)
    return init_from_pts3d(self, pts3d, im_focals, im_poses)


@torch.no_grad()
def init_from_known_poses(self, niter_PnP=10, min_conf_thr=3):
    """All camera poses and focals are given: only pairwise poses and depth maps remain to be initialised."""
    device = self.device
    n_known, known_msk, known_poses = get_known_poses(self)
    assert n_known == self.n_imgs, 'not all poses are known'
    n_focals, _, focals = get_known_focals(self)
    assert n_focals == self.n_imgs
    pps = self.get_principal_points()
    # a scene of kept rows works on the edges whose row it keeps -- all the edges (i, *) of its own images i -- and takes
    # the other pairwise poses and depth maps from their keepers
    partial = owned.shard_of(self) is not None
    mine = owned.keeps_edge(self) if partial else None
    best = {}        # image -> (score, pair key, scale) of its most confident pair
    for e, (i, j) in enumerate(self.edges):
        if partial and not mine[e]:
            continue
        key = edge_str(i, j)
        # second camera of the pair by PnP in the first camera's frame, then both onto the known cameras
        msk = self.conf_i[key] > min(min_conf_thr, self.conf_i[key].min() - 0.1)
        _, second = fast_pnp(self.pred_j[key], float(focals[i].mean()), pp=pps[i], msk=msk, device=device, niter_PnP=niter_PnP)
        s, R, T = align_multiple_poses(torch.stack((torch.eye(4, device=device), second)), known_poses[[i, j]])
        self._set_pose(self.pw_poses, e, R, T, scale=s)
        score = float(self.conf_i[key].mean())
        if score > best.get(i, (0,))[0]:
            best[i] = (score, key, s)
    for i in range(self.n_imgs):
        assert known_msk[i]
        if partial and not owned.owns_image(self, i):
            continue
        _, key, s = best[i]
        self._set_depthmap(i, self.pred_i[key][:, :, 2] * s)
    if partial:
        if self.pw_poses.requires_grad:
            owned.share_edge_rows(self, self.pw_poses)
        owned.share_image_rows(self)
