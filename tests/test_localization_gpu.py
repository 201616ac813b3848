"""localize() on the GPU (dust3r_b200.localization, the body of visloc.py:80-172 for one query):

  * with a stand-in model that serves ground-truth pointmaps through the interface inference() drives, the 2-D / 3-D
    correspondences equal, index for index, those of the reference's loop restated below (cKDTree matching on the same
    inference outputs, float64 mapping to the original pixels), and the query pose is recovered to 1e-6;
  * with the small synthetic DPT model, the one batched inference() call of localize gives the same correspondences, bit for
    bit, as the reference's batch_size=1 call per pair.
"""
import random

import numpy as np
import pytest
import torch
from PIL import Image

from dust3r_b200.utils.geometry import find_reciprocal_matches, geotrf, xy_grid

pytestmark = pytest.mark.gpu

H, W = 48, 64          # rescaled size; the original query image is twice as large


def _scene(n_maps, seed=0):
    """A query view and map views in the reference's view-dict format, all seeing a smooth non-planar surface from the query
    camera's pose (so every map pixel has the query pixel with the same 3-D point); ground-truth pointmaps in the query's
    camera frame for the stand-in model, keyed by instance."""
    rng = np.random.default_rng(seed)
    f = 60.0
    K_r = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1.0]])
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    depth = 4 + 0.5 * np.sin(xx / 7) + 0.3 * np.cos(yy / 5)
    Xc = np.stack([(xx - K_r[0, 2]) / f * depth, (yy - K_r[1, 2]) / f * depth, depth], -1)
    ang = rng.normal(size=3) * 0.2
    R = cv_rodrigues(ang)
    t = rng.normal(size=3)
    cam2world = np.eye(4)
    cam2world[:3, :3], cam2world[:3, 3] = R.T, -R.T @ t
    Xw = (Xc - t) @ R                       # world points of the query's pixels
    to_orig = np.diag([2.0, 2.0, 1.0])       # rescaled (u + 0.5) * 2 - 0.5 = original
    K_orig = np.array([[2 * f, 0, 2 * (W / 2 + 0.5) - 0.5], [0, 2 * f, 2 * (H / 2 + 0.5) - 0.5], [0, 0, 1.0]])
    # every query pixel passes the confidence threshold, so each map point's reciprocal match is its own pixel
    gt = {'0': (torch.from_numpy(Xc.astype(np.float32)), torch.full((H, W), 5.0))}
    query = dict(rgb_rescaled=torch.zeros(3, H, W), to_orig=to_orig, intrinsics=K_orig, distortion=None,
                 rgb=Image.new('RGB', (2 * W, 2 * H)), cam_to_world=cam2world)
    maps = []
    for i in range(n_maps):
        valid = torch.from_numpy(rng.uniform(size=(H, W)) > 0.2)
        maps.append(dict(rgb_rescaled=torch.zeros(3, H, W), valid_rescaled=valid, pts3d_rescaled=torch.from_numpy(Xw.astype(np.float32))))
        gt[str(1 + i)] = (torch.from_numpy(Xc.astype(np.float32)), torch.from_numpy(1 + 4 * rng.uniform(size=(H, W)).astype(np.float32)))
    return query, maps, gt


def cv_rodrigues(v):
    import cv2
    return cv2.Rodrigues(np.asarray(v, np.float64))[0]


class GroundTruthModel(torch.nn.Module):
    """Serves each view's ground-truth pointmap (query camera frame) and a fixed confidence map, by instance."""

    def __init__(self, gt):
        super().__init__()
        self.gt = gt

    def forward(self, view1, view2):
        dev = view1['img'].device
        g = lambda v, k: torch.stack([self.gt[s][k] for s in v['instance']]).to(dev)
        return dict(pts3d=g(view1, 0), conf=g(view1, 1)), dict(pts3d_in_other_view=g(view2, 0), conf=g(view2, 1))


def reference_matches(query_view, map_views, model, device, conf_thr=3.0):
    """visloc.py:80-165, restated: one inference() per pair with batch_size=1, numpy masks, cKDTree reciprocal matches."""
    from dust3r_b200.inference import inference
    q2d, q3d = [], []
    for mi, map_view in enumerate(map_views):
        imgs = []
        for idx, img in enumerate([query_view['rgb_rescaled'], map_view['rgb_rescaled']]):
            k = 0 if idx == 0 else 1 + mi
            imgs.append(dict(img=img.unsqueeze(0), true_shape=np.int32([img.shape[1:]]), idx=k, instance=str(k)))
        output = inference([tuple(imgs)], model, device, batch_size=1, verbose=False)
        pred1, pred2 = output['pred1'], output['pred2']
        confidence_masks = [pred1['conf'].squeeze(0) >= conf_thr, (pred2['conf'].squeeze(0) >= conf_thr) & map_view['valid_rescaled']]
        pts3d = [pred1['pts3d'].squeeze(0), pred2['pts3d_in_other_view'].squeeze(0)]
        pts2d_list, pts3d_list = [], []
        for i in range(2):
            conf_i = confidence_masks[i].cpu().numpy()
            true_shape_i = imgs[i]['true_shape'][0]
            pts2d_list.append(xy_grid(true_shape_i[1], true_shape_i[0])[conf_i])
            pts3d_list.append(pts3d[i].detach().cpu().numpy()[conf_i])
        PQ, PM = pts3d_list
        if len(PQ) == 0 or len(PM) == 0:
            continue
        reciprocal_in_PM, nnM_in_PQ, num_matches = find_reciprocal_matches(PQ, PM)
        matches_im1 = pts2d_list[1][reciprocal_in_PM]
        matches_im0 = pts2d_list[0][nnM_in_PQ][reciprocal_in_PM]
        valid_pts3d = map_view['pts3d_rescaled'][matches_im1[:, 1], matches_im1[:, 0]]
        matches_im0 = matches_im0.astype(np.float64) + 0.5
        matches_im0 = geotrf(query_view['to_orig'], matches_im0, norm=True) - 0.5
        if len(valid_pts3d):
            q3d.append(valid_pts3d.cpu().numpy())
            q2d.append(matches_im0)
    return np.concatenate(q2d), np.concatenate(q3d)


def test_localize_equals_reference_loop_and_recovers_pose(cuda_device):
    from dust3r_b200.localization import get_pose_error, localize, localize_matches
    query, maps, gt = _scene(4)
    model = GroundTruthModel(gt)
    p2, p3 = localize_matches(query, maps, model, cuda_device)
    r2, r3 = reference_matches(query, maps, model, cuda_device)
    assert p2.shape == r2.shape and p3.shape == r3.shape and len(r2) > 1000
    np.testing.assert_allclose(p2.cpu().numpy(), r2, rtol=0, atol=1e-12)
    assert np.array_equal(p3.cpu().numpy(), r3)
    ok, cam2world = localize(query, maps, model, cuda_device)
    assert ok
    te, ae = get_pose_error(cam2world, query['cam_to_world'])
    assert float(te) <= 1e-6 and float(ae) <= 1e-6 * 180 / np.pi, (float(te), float(ae))
    # the pnp_max_points subsample: rng.sample on the host, the reference's rows
    ok2, cam2world2 = localize(query, maps, model, cuda_device, pnp_max_points=800, rng=random.Random(3))
    assert ok2 and float(get_pose_error(cam2world2, query['cam_to_world'])[0]) <= 1e-5


def test_localize_batched_inference_equals_per_pair_calls(cuda_device):
    from test_forward_gpu import _build, _small_cfgs
    from dust3r_b200.localization import localize_matches
    from dust3r_b200.utils.synth import synth_images
    cfg, h, w = _small_cfgs()['small_dpt']
    net, _ = _build(cfg, 11, cuda_device)
    imgs = synth_images(4, h, w, seed=3)
    rng = np.random.default_rng(1)
    query = dict(rgb_rescaled=imgs[0]['img'][0], to_orig=np.diag([1.5, 1.5, 1.0]))
    maps = [dict(rgb_rescaled=im['img'][0], valid_rescaled=torch.from_numpy(rng.uniform(size=(h, w)) > 0.1),
                 pts3d_rescaled=torch.from_numpy(rng.normal(size=(h, w, 3)).astype(np.float32))) for im in imgs[1:]]
    # a confidence threshold in the range this model's confidences take, so both masks are partial
    from dust3r_b200.inference import inference
    q = dict(img=query['rgb_rescaled'][None], true_shape=np.int32([[h, w]]), idx=0, instance='0')
    out = inference([(q, dict(img=maps[0]['rgb_rescaled'][None], true_shape=np.int32([[h, w]]), idx=1, instance='1'))], net,
                    cuda_device, batch_size=1, verbose=False)
    reference_conf = float(out['pred1']['conf'].median())
    p2, p3 = localize_matches(query, maps, net, cuda_device, conf_thr=reference_conf)
    r2, r3 = reference_matches(query, maps, net, cuda_device, conf_thr=reference_conf)
    assert len(r2) > 0
    assert np.array_equal(p2.cpu().numpy(), r2) and np.array_equal(p3.cpu().numpy(), r3)
