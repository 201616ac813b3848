"""Sky segmentation kernels (csrc/sky_ops.cu, `d3r_segment_sky`) on the H100, bit-exact against oracle/sky_oracle.py run on the
same machine and against the unmodified reference's outputs (tests/golden/segment_sky.npz); mask_sky() on device scenes.  The
CPU twin (colour test on all 2^24 colours, oracle vs reference, host path) is tests/test_sky_host.py."""
import copy

import numpy as np
import pytest
import torch

from dust3r_b200.utils.synth import synth_sky_image
from oracle import sky_oracle
from test_sky_host import golden, golden_mask, sky_cases, sky_scene

pytestmark = pytest.mark.gpu


def _check(images, got):
    assert len(got) == len(images)
    for img, mask in zip(images, got):
        assert mask.is_cuda and mask.dtype == torch.bool and tuple(mask.shape) == img.shape[:2]
        assert np.array_equal(mask.cpu().numpy(), sky_oracle.segment_sky(img))


def test_every_case_alone_and_in_one_batch(cuda_device):
    from dust3r_b200 import _lib
    from dust3r_b200.cloud_opt.scene_ops import segment_sky as segment_sky_batch
    from dust3r_b200.viz import segment_sky
    gold = golden()
    cases = sky_cases()
    names = sorted(cases)
    dev_imgs = [torch.from_numpy(cases[k]).to(cuda_device) for k in names]
    for k, img in zip(names, dev_imgs):
        _lib.launch_count(reset=True)
        got = segment_sky(img)
        assert _lib.launch_count() == 7, k                 # a fixed number of launches, whatever the content
        assert got.is_cuda and got.dtype == torch.bool
        want = sky_oracle.segment_sky(cases[k])
        assert np.array_equal(want, golden_mask(gold, k)), k
        assert np.array_equal(got.cpu().numpy(), want), k
    batch = segment_sky_batch(dev_imgs)                     # every case, float and uint8, sizes mixed, in one call
    for k, got in zip(names, batch):
        assert np.array_equal(got.cpu().numpy(), golden_mask(gold, k)), k


def test_mixed_sizes_batch(cuda_device):
    from dust3r_b200.cloud_opt.scene_ops import segment_sky
    images = [synth_sky_image(h, w, seed=100 + k) for k, (h, w) in enumerate([(384, 512), (512, 384), (224, 224), (384, 512),
                                                                              (37, 53), (224, 224)])]
    _check(images, segment_sky([torch.from_numpy(x).to(cuda_device) for x in images]))


def test_fifty_images_and_determinism(cuda_device):
    from dust3r_b200 import _lib
    from dust3r_b200.cloud_opt.scene_ops import segment_sky, segment_sky_host_images
    images = [synth_sky_image(384, 512, seed=200 + k) for k in range(50)]
    dev = [torch.from_numpy(x).to(cuda_device) for x in images]
    _lib.launch_count(reset=True)
    first = segment_sky(dev)
    assert _lib.launch_count() == 7
    _check(images, first)
    second = segment_sky(dev)
    assert all(torch.equal(a, b) for a, b in zip(first, second))
    third = segment_sky_host_images(images, cuda_device)     # the pinned-upload path mask_sky takes
    assert all(torch.equal(a, b) for a, b in zip(first, third))
    assert sum(int(m.sum()) for m in first) > 0.2 * 50 * 384 * 512


def test_bad_calls_return_errors(cuda_device):
    from dust3r_b200 import _lib
    lib = _lib.get_lib()
    H, W = 64, 80
    rgb = torch.zeros((H * W * 3,), dtype=torch.uint8, device=cuda_device)
    out = torch.empty((H * W,), dtype=torch.uint8, device=cuda_device)
    hw = torch.tensor([[H, W]], dtype=torch.int32, device=cuda_device)
    off = torch.zeros((1,), dtype=torch.int64, device=cuda_device)
    need = int(lib.d3r_segment_sky_workspace_bytes(1, H * W))
    assert need >= 9 * H * W
    ws = torch.empty((need,), dtype=torch.uint8, device=cuda_device)
    stream = torch.cuda.current_stream(cuda_device).cuda_stream

    def call(n=1, max_area=H * W, total=H * W, ws_bytes=need):
        return lib.d3r_segment_sky(n, hw.data_ptr(), off.data_ptr(), max_area, total, rgb.data_ptr(), out.data_ptr(), ws.data_ptr(),
                                   ws_bytes, stream)
    assert call() == 0
    torch.cuda.synchronize()
    assert int(out.sum()) == 0
    for kw in (dict(ws_bytes=need - 1), dict(ws_bytes=0), dict(total=H * W - 1), dict(total=2 * H * W), dict(max_area=0),
               dict(n=0), dict(total=1 << 31, max_area=1 << 30, n=2)):
        assert call(**kw) != 0, kw
        with pytest.raises(_lib.D3RError, match='segment_sky'):
            _lib.check(call(**kw))
    assert lib.d3r_segment_sky_workspace_bytes(0, 10) == 0


@pytest.mark.parametrize('mode', ['PointCloudOptimizer', 'ModularPointCloudOptimizer', 'PairViewer'])
def test_mask_sky_on_device_scene(cuda_device, mode):
    from dust3r_b200.cloud_opt import GlobalAlignerMode, global_aligner
    from dust3r_b200.viz import segment_sky
    kind = 'pv' if mode == 'PairViewer' else 'pc'
    torch.manual_seed(0)
    scene = global_aligner(copy.deepcopy(sky_scene(kind)), cuda_device, mode=getattr(GlobalAlignerMode, mode), verbose=False)
    if mode != 'PairViewer':
        scene.compute_global_alignment(niter=10)
        assert scene._engine is not None
    before = [c.detach().clone() for c in scene.im_conf]
    masked = scene.mask_sky()
    n_sky = 0
    for img, c, b, m in zip(scene.imgs, masked.im_conf, before, masked.get_masks()):
        sky = segment_sky(img)                                            # host path (numpy input)
        assert c.is_cuda
        assert torch.equal(c.cpu(), torch.where(sky, torch.zeros_like(b.cpu()), b.cpu()))
        assert not m.cpu()[sky].any()
        n_sky += int(sky.sum())
    assert n_sky > 100
    for c, b in zip(scene.im_conf, before):
        assert torch.equal(c.detach(), b)
    if kind == 'pc':
        gold = golden()
        for i, c in enumerate(masked.im_conf):
            assert torch.equal(c.detach().cpu(), torch.from_numpy(gold[f'scene|pc|im_conf|{i}']))
    if mode != 'PairViewer':
        assert masked._engine is None
        loss = masked.compute_global_alignment(niter=10)
        assert np.isfinite(loss) and masked._engine is not None and masked._engine is not scene._engine
