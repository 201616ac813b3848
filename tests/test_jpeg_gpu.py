"""GPU JPEG decoder (csrc/jpeg_ops.cu) on the H100: decode_jpeg equals Pillow on the corpus of tests/test_jpeg_host.py,
load_images(device=cuda) on a mixed folder equals load_images(device=None) bit for bit with the same verbose output, inference()
on those views equals the host-loaded views', and decoding is deterministic.  Corrupt streams are only fed here when their
reads stay inside the buffer by construction (the bit reader is bounded by the byte count; the host suite checks that under
AddressSanitizer), and only their status word is checked."""
import contextlib
import io

import numpy as np
import pytest
import torch

from test_jpeg_host import (HOST_ONLY, RANGE, RANGE_CASES, _pil_jpeg, _pixels, crafted_grey_8x8, jpeg_corpus, pillow_rgb,
                             with_trailer)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def corpus():
    return jpeg_corpus()


def _device_status(data, dev):
    from dust3r_b200.utils.image import _jpeg_launch, _jpeg_stage
    staged = _jpeg_stage(data)
    assert staged is not None
    img, status = _jpeg_launch(staged, dev)
    return img, int(status.item())


def test_decode_jpeg_equals_pillow(cuda_device, corpus):
    from dust3r_b200.utils.image import decode_jpeg
    for name, data in corpus.items():
        want = pillow_rgb(data)
        got = decode_jpeg(data, cuda_device)
        assert got.device.type == 'cuda' and got.dtype == torch.uint8, name
        assert np.array_equal(got.cpu().numpy(), want), name
        if name not in HOST_ONLY:        # the kernels themselves decoded it (not the Pillow path)
            img, status = _device_status(data, cuda_device)
            assert status == 0, name
            assert np.array_equal(img.cpu().numpy(), want), name


def test_trailer_after_eoi_and_simd_range_cases(cuda_device, corpus):
    """A 1 MB trailer after EOI decodes on the device (status 0) to Pillow's pixels; the hand-built files whose IDCT outputs
    leave [-512, 511] report D3R_JPEG_RANGE, and decode_jpeg returns Pillow's pixels for them."""
    from dust3r_b200.utils.image import decode_jpeg
    for name in ('q90_420_4032x3024', 'rst7_422_1023x769'):
        data = with_trailer(corpus[name], 1 << 20)
        img, status = _device_status(data, cuda_device)
        assert status == 0 and np.array_equal(img.cpu().numpy(), pillow_rgb(data)), name
    for dc_quant, dc_coef in RANGE_CASES:
        data = crafted_grey_8x8(dc_quant, dc_coef)
        _, status = _device_status(data, cuda_device)
        assert status & RANGE, (dc_quant, dc_coef)
        assert np.array_equal(decode_jpeg(data, cuda_device).cpu().numpy(), pillow_rgb(data)), (dc_quant, dc_coef)


def test_two_decodes_are_identical(cuda_device, corpus):
    for name in ('q90_420_4032x3024', 'rst7_422_1023x769'):
        a, sa = _device_status(corpus[name], cuda_device)
        b, sb = _device_status(corpus[name], cuda_device)
        assert sa == sb == 0 and torch.equal(a, b), name


def test_corrupt_streams_report_status(cuda_device, corpus):
    """Truncated inside the scan (the buffer is the shorter file: every read stays inside it) -> non-zero status."""
    from dust3r_b200.utils import jpeg
    for name in ('q90_420_64x48', 'rst1_422_100x75', 'grey_q90_53x41'):
        data = corpus[name]
        begin = jpeg.parse(data)['scan_begin']
        for cut in (begin + 1, begin + (len(data) - begin) // 2):
            _, status = _device_status(data[:cut], cuda_device)
            assert status != 0, (name, cut)


@pytest.fixture(scope='module')
def mixed_folder(tmp_path_factory):
    import PIL.Image
    d = tmp_path_factory.mktemp('mixed')
    arr = _pixels(300, 400, 31)
    (d / 'a_baseline.jpg').write_bytes(_pil_jpeg(arr, quality=90, subsampling=2))
    (d / 'b_progressive.jpg').write_bytes(_pil_jpeg(_pixels(300, 400, 32), quality=90, progressive=True))
    (d / 'c_rotated.jpeg').write_bytes(_pil_jpeg(_pixels(240, 320, 33), quality=85, subsampling=1, orientation=6))
    (d / 'd_grey.JPG').write_bytes(_pil_jpeg(_pixels(320, 256, 34), mode='L', quality=80))
    PIL.Image.fromarray(_pixels(200, 280, 35)).save(d / 'e_image.png')
    (d / 'f_restart.jpg').write_bytes(_pil_jpeg(_pixels(288, 384, 36), quality=95, subsampling=0, restart_marker_blocks=5))
    (d / 'g_notes.txt').write_text('skipped')
    return str(d)


def _load(folder, device, workers):
    from dust3r_b200.utils.image import load_images
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        views = load_images(folder, size=224 if workers == 3 else 512, device=device, workers=workers)
    return views, buf.getvalue()


@pytest.mark.parametrize('workers', [1, 3, 4])
def test_load_images_device_equals_host(cuda_device, mixed_folder, workers):
    host, host_log = _load(mixed_folder, None, workers)
    dev, dev_log = _load(mixed_folder, cuda_device, workers)
    assert dev_log == host_log and len(host) == 6
    for h, d in zip(host, dev):
        assert d['img'].device.type == 'cuda'
        assert torch.equal(d['img'].cpu(), h['img']), h['idx']
        assert np.array_equal(d['true_shape'], h['true_shape']) and d['idx'] == h['idx'] and d['instance'] == h['instance']


def test_inference_on_device_loaded_views_equals_host_loaded(cuda_device, mixed_folder):
    from dust3r_b200.image_pairs import make_pairs
    from dust3r_b200.inference import inference
    from dust3r_b200.model import AsymmetricCroCo3DStereo
    from dust3r_b200.utils.synth import synth_state_dict
    from dust3r_b200.config import ModelConfig
    cfg = ModelConfig(img_size=(224, 224), enc_embed_dim=128, enc_depth=2, enc_num_heads=2, dec_embed_dim=128, dec_depth=2,
                      dec_num_heads=2, head_type='linear', landscape_only=False)
    model = AsymmetricCroCo3DStereo(pos_embed='RoPE100', img_size=cfg.img_size, head_type='linear', enc_embed_dim=128,
                                    enc_depth=2, enc_num_heads=2, dec_embed_dim=128, dec_depth=2, dec_num_heads=2,
                                    landscape_only=False)
    model.load_state_dict(synth_state_dict(cfg, seed=3))
    model = model.to(cuda_device).eval()
    outs = []
    for device in (None, cuda_device):
        views, _ = _load(mixed_folder, device, 3)
        pairs = make_pairs(views, scene_graph='complete', symmetrize=True)
        outs.append(inference(pairs, model, cuda_device, batch_size=4, verbose=False))
    for view in ('pred1', 'pred2'):
        for key in outs[0][view]:
            a, b = outs[0][view][key], outs[1][view][key]
            if torch.is_tensor(a):
                assert torch.equal(a.cpu(), b.cpu()), (view, key)
