"""The view stage on the CPU (dust3r_b200.views): the host plan and port against the reference's BaseStereoViewDataset
(tests/golden/views.npz, made by tests/golden/make_views_golden.py from the unmodified reference) and against the CPU oracle
(oracle/views_oracle.py), RNG state included; the per-thread bodies of the CUDA kernels (csrc/view_core.h) compiled with g++ and
run over every block and thread of the three launches, bit-equal to the oracle; and the inputs the stage rejects."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
import native_harness

from dust3r_b200.utils.synth import synth_rgbd_frame
from dust3r_b200.views import final_crop_box, item_rng, prepare_batch, prepare_views, view_descriptors
from oracle.views_oracle import digest, views_oracle

PIXELS = ('img', 'depthmap', 'pts3d', 'valid_mask')


def golden():
    return np.load(os.path.join(GOLDEN, 'views.npz'))


def golden_cases():
    return json.loads(str(golden()['cases']))


def case_frames(case):
    return [synth_rgbd_frame(**spec) for spec in case['frames']]


def case_rng(case):
    return item_rng(case['seed'], case['idx'])


def check_golden(case, views, G=None):
    """The views of `case` (any producer: numpy arrays or tensors on any device) equal the reference's, bit for bit."""
    G = golden() if G is None else G
    assert len(views) == len(case['frames'])
    for v, view in enumerate(views):
        key = f'{case["name"]}|{v}|'
        for k in PIXELS:
            assert digest(view[k]) == str(G[key + k]), (case['name'], v, k)
        for k in ('camera_intrinsics', 'camera_pose', 'true_shape'):
            got = view[k].cpu().numpy() if torch.is_tensor(view[k]) else np.asarray(view[k])
            assert got.dtype == G[key + k].dtype and np.array_equal(got, G[key + k], equal_nan=k == 'camera_pose'), (case['name'], v, k)
        assert tuple(view['idx']) == tuple(int(i) for i in G[key + 'idx']), (case['name'], v)
        assert view['rng'] == int(G[key + 'rng']), (case['name'], v)


def equal_nan(a, b):
    """Bit-equal up to NaN payloads (NaN-aware torch.equal)."""
    a, b = torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).cpu(), torch.as_tensor(np.asarray(b) if not torch.is_tensor(b) else b).cpu()
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.is_floating_point():
        na, nb = torch.isnan(a), torch.isnan(b)
        return torch.equal(na, nb) and torch.equal(a[~na], b[~nb])
    return torch.equal(a, b)


@pytest.mark.parametrize('case', golden_cases(), ids=lambda c: c['name'])
def test_oracle_equals_reference_golden(case):
    check_golden(case, views_oracle(case_frames(case), case['resolution'], case_rng(case), idx=case['idx'],
                                    aug_crop=case.get('aug_crop', False)))


@pytest.mark.parametrize('case', golden_cases(), ids=lambda c: c['name'])
def test_host_port_equals_golden_and_oracle(case):
    frames = case_frames(case)
    rng, orng = case_rng(case), case_rng(case)
    views = prepare_views(frames, tuple(case['resolution']), rng=rng, idx=case['idx'], aug_crop=case.get('aug_crop', False),
                          device='cpu')
    check_golden(case, views)
    want = views_oracle(frames, case['resolution'], orng, idx=case['idx'], aug_crop=case.get('aug_crop', False))
    assert rng.bit_generator.state == orng.bit_generator.state
    for got, ref in zip(views, want):
        for k in PIXELS + ('camera_intrinsics',):
            assert equal_nan(got[k], ref[k]), k


def test_near_square_draws_both_orientations():
    G = golden()
    shapes = {tuple(G[f'{name}|{v}|true_shape']) for name in ('near_square', 'near_square_b') for v in range(2)}
    assert shapes == {(384, 512), (512, 384)}


@pytest.mark.skipif(not os.environ.get('DUST3R_REFERENCE'), reason='DUST3R_REFERENCE not set')
def test_oracle_equals_live_reference():
    import sys
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    from make_views_golden import CASES, SynthFrames
    for case in CASES:
        ds = SynthFrames(case['frames'], resolution=tuple(case['resolution']), aug_crop=case.get('aug_crop', False), seed=case['seed'])
        ref = ds[case['idx']]
        got = views_oracle(case_frames(case), case['resolution'], case_rng(case), idx=case['idx'], aug_crop=case.get('aug_crop', False))
        for r, g in zip(ref, got):
            for k in PIXELS + ('camera_intrinsics', 'camera_pose', 'true_shape'):
                assert equal_nan(r[k], g[k]), (case['name'], k)
            assert r['rng'] == g['rng'] and r['idx'] == g['idx']


# ------------------------------------------------------------------------------------------------------------------
# csrc/view_core.h on the host
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def view_host():
    lib = ctypes.CDLL(native_harness.build('view_host'))
    lib.view_host.restype = ctypes.c_int
    lib.view_host.argtypes = [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]
    return lib


# (H, W, seed, pose) of the frames run through the harness in one call: landscape / portrait / near-square, down- and up-scaled,
# odd sizes, an off-centre principal point, no pose
NATIVE_FRAMES = [(480, 640, 1, True), (640, 480, 2, True), (520, 500, 3, True), (500, 510, 4, True), (150, 200, 5, True),
                 (160, 120, 6, True), (1000, 700, 7, True), (333, 517, 8, True), (517, 333, 9, True), (384, 512, 10, True),
                 (768, 1024, 11, True), (97, 131, 12, True), (1201, 901, 13, True), (480, 640, 14, False), (721, 1283, 15, True)]


def fill_table_cache(monkeypatch, n):
    """The shared coefficient-table cache of dust3r_b200.utils.image holding `n` entries of other images (it is cleared when
    it passes 512 entries), restored after the test."""
    from dust3r_b200.utils import image
    monkeypatch.setattr(image, '_DEVICE_TABLES', {('other image', i): None for i in range(n)})


def test_view_desc_mirror_matches_the_library():
    from dust3r_b200 import _lib
    assert ctypes.sizeof(_lib.ViewDesc) == _lib.get_lib().d3r_sizeof_view_desc()


@pytest.mark.parametrize('resolution,aug_crop,cached', [((512, 384), False, 0), ((512, 288), 8, 0), ((224, 224), False, 0),
                                                        ((224, 224), False, 505)])
def test_native_view_core_equals_oracle(view_host, monkeypatch, resolution, aug_crop, cached):
    """With cached=505 the shared table cache is cleared a few views into the call: the descriptors must still point at
    live tables."""
    from dust3r_b200.utils.image import norm_lut
    from dust3r_b200.views import _empty_outputs, _plan_item
    fill_table_cache(monkeypatch, cached)
    frames = [synth_rgbd_frame(H, W, seed, pose=pose, pp=(0.31 * W, 0.55 * H) if seed == 8 else None)
              for H, W, seed, pose in NATIVE_FRAMES]
    plans = _plan_item(frames, resolution, np.random.default_rng(5), aug_crop)
    want = views_oracle(frames, resolution, np.random.default_rng(5), aug_crop=aug_crop)
    cpu = torch.device('cpu')
    outs = [_empty_outputs(p, cpu) for p in plans]
    for out in outs:
        for t in out.values():
            t.view(torch.uint8).fill_(0xA5)      # garbage: every element must be written
    descs, keep = view_descriptors(frames, plans, outs, cpu)
    from dust3r_b200.utils import image
    assert not cached or len(image._DEVICE_TABLES) < cached      # the cache was cleared during the call
    lut = norm_lut()
    assert view_host.view_host(len(frames), ctypes.addressof(descs), lut.data_ptr()) == 0
    for i, (out, ref) in enumerate(zip(outs, want)):
        for k in PIXELS:
            assert equal_nan(out[k], ref[k]), (NATIVE_FRAMES[i], k)


# ------------------------------------------------------------------------------------------------------------------
# batches, draws, rejections
# ------------------------------------------------------------------------------------------------------------------
def _oracle_batch(items, resolution, seed=None, rng=None):
    from torch.utils.data import default_collate
    out = []
    for idx, frames in items:
        r = item_rng(seed, idx) if seed else rng
        views = views_oracle(frames, resolution, r, idx=idx)
        for f, view in zip(frames, views):
            view.update({k: f[k] for k in ('dataset', 'label', 'instance')})
        out.append(views)
    return default_collate(out)


@pytest.mark.parametrize('mode', ['seed', 'rng'])
def test_prepare_batch_cpu_equals_collated_oracle(mode):
    items = []
    for b, (H, W) in enumerate([(480, 640), (640, 480), (505, 500), (150, 200)]):
        frames = [synth_rgbd_frame(H, W, 40 + 2 * b), synth_rgbd_frame(W, H, 41 + 2 * b, pose=b != 1)]
        for v, f in enumerate(frames):
            f.update(dataset='synth', label=f'scene{b}', instance=f'{b}_{v}')
        items.append((10 + b, frames))
    kw = dict(seed=3) if mode == 'seed' else dict(rng=np.random.default_rng(9))
    ref = _oracle_batch(items, (512, 384), **(dict(seed=3) if mode == 'seed' else dict(rng=np.random.default_rng(9))))
    got = prepare_batch(items, (512, 384), device='cpu', **kw)
    for g, r in zip(got, ref):
        assert set(g) == set(r)
        for k in r:
            if torch.is_tensor(r[k]):
                assert equal_nan(g[k], r[k]), k
            elif k == 'idx':
                assert all(torch.equal(a, b) for a, b in zip(g[k], r[k]))
            else:
                assert g[k] == r[k], k


def _frame(**changes):
    f = synth_rgbd_frame(96, 128, 1)
    f.update(changes)
    return f


@pytest.mark.parametrize('bad,match', [
    (dict(depthmap=np.where(np.eye(96, 128, dtype=bool), np.float32(np.nan), synth_rgbd_frame(96, 128, 1)['depthmap'])), 'non-finite depth'),
    (dict(depthmap=np.full((96, 128), np.inf, dtype=np.float32)), 'non-finite depth'),
    (dict(camera_pose=np.full((4, 4), np.nan, dtype=np.float32)), 'non-finite camera_pose'),
    (dict(camera_intrinsics=np.array([[100, 0.5, 64], [0, 100, 48], [0, 0, 1]], dtype=np.float32)), 'skewed'),
    (dict(camera_intrinsics=np.array([[100, 0, 64], [0, 100, 48], [0, 0, 1]], dtype=np.float64)), 'float32 3x3'),
    (dict(camera_intrinsics=np.array([[100, 0, 200], [0, 100, 48], [0, 0, 1]], dtype=np.float32)), 'principal point'),
    (dict(depthmap=np.ones((96, 128), dtype=np.float64)), 'depthmap must be float32'),
    (dict(img=np.zeros((96, 128, 4), dtype=np.uint8)), 'img must be uint8'),
])
def test_rejections(bad, match):
    with pytest.raises(ValueError, match=match):
        prepare_views([_frame(), _frame(**bad)], (512, 384), rng=np.random.default_rng(0), device='cpu')


def test_depth_is_checked_where_the_view_samples_it():
    """Like the reference, which asserts on the view's depth map: non-finite depth outside the principal-point crop, or on
    pixels the nearest-neighbour resize skips, is accepted (and changes nothing); on a sampled pixel it is refused."""
    frame = synth_rgbd_frame(960, 1280, 3, pp=(640.0, 480.0))      # crop = whole frame, 1280 -> 512: source 0, 2, 5, 7, ...
    clean = prepare_views([frame, frame], (512, 384), rng=np.random.default_rng(0), device='cpu')
    holes = dict(frame, depthmap=frame['depthmap'].copy())
    holes['depthmap'][1, 1] = np.nan
    holes['depthmap'][4, 3] = np.inf
    got = prepare_views([holes, frame], (512, 384), rng=np.random.default_rng(0), device='cpu')
    want = views_oracle([holes, frame], (512, 384), np.random.default_rng(0))
    for g, c, w in zip(got, clean, want):
        for k in PIXELS:
            assert equal_nan(g[k], c[k]) and equal_nan(g[k], w[k]), k
    off = synth_rgbd_frame(96, 128, 1, pp=(38.4, 48.0))            # crop = columns [0, 76)
    off['depthmap'][:, 100:] = np.nan
    prepare_views([off, off], (512, 384), rng=np.random.default_rng(0), device='cpu')
    holes['depthmap'][2, 2] = np.nan
    with pytest.raises(ValueError, match='view 0: non-finite depth'):
        prepare_views([holes, frame], (512, 384), rng=np.random.default_rng(0), device='cpu')
    with pytest.raises(ValueError, match='item 7 view 1: non-finite depth'):
        prepare_batch([(6, [frame, frame]), (7, [frame, holes])], (512, 384), rng=np.random.default_rng(0), device='cpu')


def test_final_crop_box_leaving_the_image_is_rejected():
    K = np.array([[100, 0, 40], [0, 100, 30], [0, 0, 1]], dtype=np.float32)
    assert final_crop_box(K, K, (64, 48), (64, 48)) == (0, 0, 64, 48)
    shifted = K.copy()
    shifted[0, 2] = 37
    assert final_crop_box(K, shifted, (64, 48), (67, 48)) == (3, 0, 67, 48)
    with pytest.raises(ValueError, match='leaves the resized'):
        final_crop_box(K, shifted, (64, 48), (66, 48))
    shifted[1, 2] = 31
    with pytest.raises(ValueError, match='leaves the resized'):
        final_crop_box(K, shifted, (64, 48), (64, 48))


def test_bad_resolution_and_missing_rng():
    f = _frame()
    with pytest.raises(ValueError, match='resolution'):
        prepare_views([f, f], (384, 512), rng=np.random.default_rng(0), device='cpu')
    with pytest.raises(ValueError, match='Generator'):
        prepare_views([f, f], (512, 384), rng=None, device='cpu')
    with pytest.raises(ValueError, match='Generator'):
        prepare_batch([(0, [f, f])], (512, 384), device='cpu')
