"""The view stage on the H100 (d3r_prepare_views, csrc/view_ops.cu, behind dust3r_b200.views): every reference case alone and
all of them in one call bit-equal to the reference's golden and to the host port, frames decoded on the device read in place,
large frames, repeat calls, descriptors the library must refuse, and loss_of_one_batch on device-prepared batches equal to
host-prepared ones."""
import ctypes

import numpy as np
import pytest
import torch

from dust3r_b200.utils.synth import synth_rgbd_frame
from dust3r_b200.views import item_rng, prepare_batch, prepare_views

from test_views_host import PIXELS, case_frames, case_rng, check_golden, equal_nan, fill_table_cache, golden, golden_cases

pytestmark = pytest.mark.gpu


def _same(got, want, keys=PIXELS + ('camera_intrinsics', 'camera_pose', 'true_shape')):
    for g, w in zip(got, want):
        for k in keys:
            assert equal_nan(g[k], w[k]), k
        assert g['rng'] == w['rng'] and g['idx'] == w['idx']


@pytest.mark.parametrize('case', golden_cases(), ids=lambda c: c['name'])
def test_case_equals_golden_and_host(case, cuda_device):
    kw = dict(idx=case['idx'], aug_crop=case.get('aug_crop', False))
    rng = case_rng(case)
    got = prepare_views(case_frames(case), tuple(case['resolution']), rng=rng, device=cuda_device, **kw)
    assert all(v[k].device == cuda_device for v in got for k in PIXELS)
    check_golden(case, got)
    host_rng = case_rng(case)
    _same(got, prepare_views(case_frames(case), tuple(case['resolution']), rng=host_rng, device='cpu', **kw))
    assert rng.bit_generator.state == host_rng.bit_generator.state


@pytest.mark.parametrize('cached', [0, 505])
def test_all_cases_in_one_call(cuda_device, monkeypatch, cached):
    """Every golden case of one resolution as one batch, one d3r_prepare_views call (three launches) for all its views of
    mixed sizes, orientations and scales, with and without pose: each view equals the golden.  prepare_batch(seed=1) draws
    item i from default_rng(1 + i), so item idx = case seed + case idx - 1 makes each case draw what it drew alone.  With
    cached=505 the shared coefficient-table cache is cleared partway through the call."""
    from dust3r_b200 import _lib
    fill_table_cache(monkeypatch, cached)
    G = golden()
    cases = [c for c in golden_cases() if c['resolution'] == [512, 384] and not c.get('aug_crop')]
    items = [(c['seed'] + c['idx'] - 1, case_frames(c)) for c in cases]
    n0 = _lib.launch_count()
    view1, view2 = prepare_batch(items, (512, 384), seed=1, device=cuda_device)
    assert _lib.launch_count() - n0 == 3
    for b, case in enumerate(cases):
        per_view = []
        for v, view in enumerate((view1, view2)):
            pv = {k: view[k][b] for k in PIXELS + ('camera_intrinsics', 'camera_pose', 'true_shape')}
            pv.update(idx=(case['idx'], 0, v), rng=int(view['rng'][b]))
            assert [int(t[b]) for t in view['idx']] == [items[b][0], 0, v]
            per_view.append(pv)
        check_golden(case, per_view, G)


def test_device_depth_checked_where_sampled(cuda_device):
    """Non-finite depth the view never samples is accepted, a sampled one refused, for depth maps already on the device."""
    frame = synth_rgbd_frame(960, 1280, 3, pp=(640.0, 480.0))      # crop = whole frame, 1280 -> 512: source 0, 2, 5, 7, ...
    depth = torch.from_numpy(frame['depthmap']).to(cuda_device)
    holes = dict(frame, depthmap=depth.clone())
    holes['depthmap'][1, 1] = float('nan')
    got = prepare_views([holes, frame], (512, 384), rng=np.random.default_rng(0), device=cuda_device)
    _same(got, prepare_views([frame, frame], (512, 384), rng=np.random.default_rng(0), device=cuda_device))
    holes['depthmap'][2, 2] = float('inf')
    with pytest.raises(ValueError, match='item 4 view 0: non-finite depth'):
        prepare_batch([(4, [holes, frame])], (512, 384), rng=np.random.default_rng(0), device=cuda_device)


def test_device_frames_read_in_place(cuda_device):
    """Frames from decode_jpeg (and depth maps already in HBM) go in without a host round trip and give the host port's bits."""
    import io
    import PIL.Image
    from dust3r_b200.utils.image import decode_jpeg
    frames = []
    for H, W, seed in [(480, 640, 1), (900, 600, 2)]:
        f = synth_rgbd_frame(H, W, seed)
        buf = io.BytesIO()
        PIL.Image.fromarray(f['img']).save(buf, 'JPEG', quality=90)
        f['img'] = decode_jpeg(buf.getvalue(), cuda_device)
        f['depthmap'] = torch.from_numpy(f['depthmap']).to(cuda_device)
        frames.append(f)
    ptrs = [f['img'].data_ptr() for f in frames]
    got = prepare_views(frames, (512, 384), rng=item_rng(5, 1), idx=1, device=cuda_device)
    assert [f['img'].data_ptr() for f in frames] == ptrs
    _same(got, prepare_views(frames, (512, 384), rng=item_rng(5, 1), idx=1, device='cpu'))


@pytest.mark.timeout(900)
def test_large_frames_and_repeat_calls(cuda_device):
    frames = [synth_rgbd_frame(3024, 4032, 1), synth_rgbd_frame(1440, 1920, 2)]
    got = prepare_views(frames, (512, 384), rng=item_rng(1, 0), device=cuda_device)
    again = prepare_views(frames, (512, 384), rng=item_rng(1, 0), device=cuda_device)
    for g, a in zip(got, again):
        for k in PIXELS:
            assert torch.equal(g[k].nan_to_num(), a[k].nan_to_num()), k
    _same(got, prepare_views(frames, (512, 384), rng=item_rng(1, 0), device='cpu'))


def test_bad_descriptors_are_refused(cuda_device):
    from dust3r_b200 import _lib, views
    from dust3r_b200.utils.image import device_lut
    f = synth_rgbd_frame(96, 128, 1)
    plans = views._plan_item([f], (64, 48), np.random.default_rng(0), False)
    outs = [views._empty_outputs(plans[0], cuda_device)]
    descs, keep = views.view_descriptors([f], plans, outs, cuda_device)
    desc_dev = torch.empty((4 * ctypes.sizeof(_lib.ViewDesc),), dtype=torch.uint8, device=cuda_device)
    lut = device_lut(cuda_device)
    run = lambda n, d: _lib.launch(cuda_device, 'd3r_prepare_views', n, d, desc_dev.data_ptr(), lut.data_ptr())  # noqa: E731
    run(1, descs)
    good = bytes(descs)
    for field, value, match in [('crop_x0', 10 ** 6, 'leaves the resized'), ('crop_y0', -1, 'leaves the resized'),
                                ('rows', 10 ** 6, 'source rows'), ('row0', -3, 'source rows'), ('W2', 0, 'positive'),
                                ('src_pitch', 1, 'pitch'), ('img', None, 'null pointer'), ('tmp', None, 'null pointer')]:
        bad = (_lib.ViewDesc * 1).from_buffer_copy(good)
        setattr(bad[0], field, value)
        with pytest.raises(_lib.D3RError, match=match):
            run(1, bad)
    with pytest.raises(_lib.D3RError, match='n_views'):
        run(0, descs)
    torch.cuda.synchronize()


@pytest.mark.timeout(900)
def test_loss_of_one_batch_device_equals_host_prepared(cuda_device):
    import dust3r_b200.losses as L
    from dust3r_b200.inference import loss_of_one_batch
    from test_forward_gpu import _build, _small_cfgs
    cfg, H, W = _small_cfgs()['small_dpt']
    net, _ = _build(cfg, 5, cuda_device)
    items = [(b, [dict(synth_rgbd_frame(h + 8 * v, w, 60 + 2 * b + v), dataset='synth', label=str(b), instance=f'{b}_{v}')
                  for v in range(2)])
             for b, (h, w) in enumerate([(480, 640), (300, 400), (120, 150), (600, 1000)])]
    crit = L.ConfLoss(L.Regr3D(L.L21, norm_mode='avg_dis'), alpha=0.2)
    losses = []
    for device in (cuda_device, 'cpu'):
        batch = prepare_batch(items, (W, H), seed=777, device=device)
        with torch.no_grad():
            loss, details = loss_of_one_batch(batch, net, crit, cuda_device, symmetrize_batch=True)['loss']
        losses.append((loss.cpu(), details))
    assert torch.equal(losses[0][0], losses[1][0]) and losses[0][1] == losses[1][1]
    assert torch.isfinite(losses[0][0])
