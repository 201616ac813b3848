"""SURVEY §8f rows as CUDA kernels (csrc/scene_ops.cu) against their fp32 host ports: clean_pointcloud, weighted Procrustes,
Weiszfeld focal, reciprocal nearest neighbours.  The host ports of clean_pointcloud and the Weiszfeld focal are pinned against
the reference (tests/golden/scene_ops.npz) only through the float64 oracle in tests/test_scene_float64_host.py; the element-by-
element kernel checks against that oracle are in tests/test_scene_float64_gpu.py."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _scene(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    f = 1.1 * max(H, W)
    K = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], dtype=torch.float32).repeat(n, 1, 1)
    cams, pts, depth, conf = [], [], [], []
    vs, us = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing='ij')
    for i in range(n):
        ang = 0.2 * (i - (n - 1) / 2)
        R = torch.tensor([[math.cos(ang), 0, math.sin(ang)], [0, 1, 0], [-math.sin(ang), 0, math.cos(ang)]], dtype=torch.float32)
        t = torch.tensor([0.8 * math.sin(ang), 0.03 * i, 0.1 * (1 - math.cos(ang))])
        c2w = torch.eye(4)
        c2w[:3, :3], c2w[:3, 3] = R, t
        d = 2.0 + torch.nn.functional.interpolate(torch.rand((1, 1, 5, 5), generator=g), size=(H, W), mode='bicubic', align_corners=True)[0, 0]
        d = d + 0.3 * torch.rand((H, W), generator=g)      # rough surfaces: plenty of see-through contradictions
        cam_pts = torch.stack(((us - W / 2) * d / f, (vs - H / 2) * d / f, d), dim=-1)
        pts.append(cam_pts @ R.T + t)
        depth.append(d)
        conf.append(1 + 3 * torch.rand((H, W), generator=g))
        cams.append(torch.linalg.inv(c2w))
    return K, torch.stack(cams), depth, pts, conf


def test_clean_pointcloud_kernel_matches_host_port(cuda_device):
    from dust3r_b200.cloud_opt.pointcloud_filter import clean_pointcloud
    n, H, W = 5, 48, 64
    K, cams, depth, pts, conf = _scene(n, H, W, seed=3)
    ref = clean_pointcloud(conf, K, cams, depth, pts, tol=0.001, bad_conf=0)            # CPU tensors -> torch host port
    dev = cuda_device
    got = clean_pointcloud([c.to(dev) for c in conf], K.to(dev), cams.to(dev), [d.to(dev) for d in depth], [p.to(dev) for p in pts],
                           tol=0.001, bad_conf=0)
    changed = sum(int((r != c).sum()) for r, c in zip(ref, conf))
    assert changed > 100                                       # the scenario does cut confidences
    bad = sum(int((g.cpu() != r).sum()) for g, r in zip(got, ref))
    assert bad <= max(2, changed // 500), (bad, changed)       # borderline pixels (rounding of the projection) only
    # mixed image sizes (ModularPointCloudOptimizer scenes)
    conf2 = [conf[0], conf[1][:32, :48].contiguous()]
    depth2 = [depth[0], depth[1][:32, :48].contiguous()]
    pts2 = [pts[0], pts[1][:32, :48].contiguous()]
    ref2 = clean_pointcloud(conf2, K[:2], cams[:2], depth2, pts2)
    got2 = clean_pointcloud([c.to(dev) for c in conf2], K[:2].to(dev), cams[:2].to(dev), [d.to(dev) for d in depth2], [p.to(dev) for p in pts2])
    assert sum(int((g.cpu() != r).sum()) for g, r in zip(got2, ref2)) <= 2


def test_weighted_procrustes_kernel_matches_host_port(cuda_device):
    from dust3r_b200.cloud_opt.commons import rigid_points_registration
    g = torch.Generator().manual_seed(5)
    for P in (1000, 384 * 512):
        x = torch.randn((P, 3), generator=g) * torch.tensor([2.0, 1.0, 0.5]) + torch.tensor([0.3, -1.0, 4.0])
        q = torch.randn(4, generator=g)
        q = q / q.norm()
        w_, xq, yq, zq = q.tolist()
        R = torch.tensor([[1 - 2 * (yq * yq + zq * zq), 2 * (xq * yq - zq * w_), 2 * (xq * zq + yq * w_)],
                          [2 * (xq * yq + zq * w_), 1 - 2 * (xq * xq + zq * zq), 2 * (yq * zq - xq * w_)],
                          [2 * (xq * zq - yq * w_), 2 * (yq * zq + xq * w_), 1 - 2 * (xq * xq + yq * yq)]])
        y = 1.7 * x @ R.T + torch.tensor([0.5, 2.0, -1.0]) + 0.01 * torch.randn((P, 3), generator=g)
        w = 1 + 5 * torch.rand((P,), generator=g)
        Rr, tr, sr = rigid_points_registration(x.double(), y.double(), weights=w.double(), compute_scaling=True)   # fp64 host port
        Rg, tg, sg = rigid_points_registration(x.to(cuda_device), y.to(cuda_device), weights=w.to(cuda_device), compute_scaling=True)
        assert float((Rg.cpu().double() - Rr).abs().max()) < 2e-6
        assert float((tg.cpu().double() - tr).abs().max()) < 2e-5
        assert abs(float(sg) - float(sr)) < 2e-6 * float(sr)
        assert abs(float(sr) - 1.7) < 1e-2
    # batched form
    xb = torch.randn((3, 500, 3), generator=g)
    yb = 0.5 * xb + 1
    wb = torch.rand((3, 500), generator=g) + 0.1
    Rg, tg, sg = rigid_points_registration(xb.to(cuda_device), yb.to(cuda_device), weights=wb.to(cuda_device), compute_scaling=True)
    assert Rg.shape == (3, 3, 3) and float((Rg.cpu() - torch.eye(3)).abs().max()) < 1e-5 and float((sg.cpu() - 0.5).abs().max()) < 1e-5


def test_weiszfeld_focal_kernel_matches_host_port(cuda_device):
    from dust3r_b200.post_process import estimate_focal_knowing_depth
    g = torch.Generator().manual_seed(7)
    B, H, W = 3, 96, 128
    vs, us = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing='ij')
    pts = []
    for f in (90.0, 140.0, 210.0):
        d = 1.5 + torch.rand((H, W), generator=g)
        p = torch.stack(((us - W / 2) * d / f, (vs - H / 2) * d / f, d), dim=-1)
        p = p + 0.02 * torch.randn(p.shape, generator=g)
        p[0, 0] = torch.tensor([0.0, 0.0, 0.0])        # a degenerate pixel: 0/0 rays are ignored
        pts.append(p)
    pts = torch.stack(pts)
    pp = torch.tensor([[W / 2, H / 2]]).repeat(B, 1)
    ref = estimate_focal_knowing_depth(pts, pp, focal_mode='weiszfeld')
    got = estimate_focal_knowing_depth(pts.to(cuda_device), pp.to(cuda_device), focal_mode='weiszfeld').cpu()
    assert torch.allclose(got, ref, rtol=2e-4), (got, ref)
    assert abs(float(ref[1]) - 140.0) < 3.0


def test_reciprocal_matches_kernel_matches_kdtree(cuda_device):
    from dust3r_b200.utils.geometry import find_reciprocal_matches
    g = torch.Generator().manual_seed(9)
    P1 = torch.randn((5000, 3), generator=g)
    P2 = torch.cat((P1[:3000] + 0.01 * torch.randn((3000, 3), generator=g), torch.randn((1500, 3), generator=g)))
    m_ref, nn_ref, cnt_ref = find_reciprocal_matches(P1.numpy(), P2.numpy())
    m, nn, cnt = find_reciprocal_matches(P1.to(cuda_device), P2.to(cuda_device))
    assert cnt == int(cnt_ref) and cnt > 2000
    assert np.array_equal(m.cpu().numpy(), m_ref) and np.array_equal(nn.cpu().numpy(), nn_ref)


def test_mst_init_on_device_recovers_consistent_scene(cuda_device):
    """init='mst' with the scene resident on the GPU: pairwise Procrustes (weighted Umeyama) and the Weiszfeld focal run through
    the CUDA kernels; the recovered focals / relative camera geometry must match the ground truth of a consistent scene, and the
    first alignment loss must be far below the uninitialised one."""
    import copy
    import cv2
    from dust3r_b200.cloud_opt import global_aligner
    from dust3r_b200.utils.synth import synth_consistent_scene
    n, H, W = 4, 48, 64
    edges = [(i, j) for i in range(n) for j in range(n) if i != j]
    out, cams, f = synth_consistent_scene(n, edges, H, W, seed=1, noise=0.0)
    for side, key in (('pred1', 'pts3d'), ('pred1', 'conf'), ('pred2', 'pts3d_in_other_view'), ('pred2', 'conf')):
        out[side][key] = out[side][key].to(cuda_device)
    cv2.setRNGSeed(0)
    torch.manual_seed(0)
    net = global_aligner(copy.deepcopy(out), cuda_device, verbose=False)
    loss_cold = float(net.forward())
    net.compute_global_alignment(init='mst', niter=0)
    loss_init = float(net.forward())
    assert loss_init < 0.2 * loss_cold, (loss_init, loss_cold)
    focals = net.get_focals().detach().cpu().reshape(-1)
    assert all(abs(float(fo) - f) / f < 0.05 for fo in focals), (focals, f)
    c_est = net.get_im_poses().detach().cpu()[:, :3, 3]
    c_gt = cams[:, :3, 3]
    d_est, d_gt = torch.cdist(c_est, c_est), torch.cdist(c_gt, c_gt)
    s = d_est.sum() / d_gt.sum()
    assert torch.allclose(d_est, s * d_gt, atol=0.05 * float(d_gt.max()) * float(s))
