"""GPU PNG decoder (csrc/png_ops.cu) on the H100: decode_png equals Pillow on the corpus of tests/test_png_host.py (a 4032x3024
file included), load_images(device=cuda) on a folder mixing JPEG and PNG kinds (every PNG routed to the GPU) equals load_images(device=None)
bit for bit with the same verbose output, large PNGs take the GPU path by default, inference() reads the PNG-loaded views in place, and decoding is deterministic.  Corrupt streams
are fed here only where every read stays inside the buffer by construction (the bit reader is bounded by the byte count; the
host suite checks that under AddressSanitizer), and only their status word is checked."""
import numpy as np
import pytest
import torch

from test_jpeg_gpu import _load
from test_jpeg_host import _pil_jpeg, _pixels
from test_png_host import (crafted_streams, excluded_files, exif_bytes, pil_png, pillow_rgb, pixels, png_corpus,
                           raw_png)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def corpus():
    return png_corpus()


def _device_status(data, dev):
    from dust3r_b200.utils.image import _png_launch, _png_stage
    staged = _png_stage(data)
    assert staged is not None
    img, status = _png_launch(staged, dev)
    return img, int(status.item())


def test_decode_png_equals_pillow(cuda_device, corpus):
    """Every file through the kernels themselves (status 0) and through decode_png, byte for byte."""
    from dust3r_b200.utils.image import decode_png
    for name, data in corpus.items():
        want = pillow_rgb(data)
        img, status = _device_status(data, cuda_device)
        assert status == 0, (name, status)
        assert np.array_equal(img.cpu().numpy(), want), name
        got = decode_png(data, cuda_device)
        assert got.device.type == 'cuda' and got.dtype == torch.uint8, name
        assert np.array_equal(got.cpu().numpy(), want), name


def test_refused_and_excluded_files_give_pillows_result(cuda_device):
    """Crafted streams report their status bit and decode_png returns Pillow's pixels (or raises what Pillow raises); files
    outside the set go to Pillow from their header."""
    from dust3r_b200.utils.image import decode_png
    cases = [(name, data, bit) for name, (data, bit) in crafted_streams().items()]
    cases += [(name, data, None) for name, (data, why) in excluded_files().items() if why is not None]
    for name, data, bit in cases:
        if bit is not None:
            _, status = _device_status(data, cuda_device)
            assert status & bit, (name, status)
        try:
            want = pillow_rgb(data)
        except Exception as e:                                  # noqa: BLE001 -- decode_png must raise what Pillow raises
            with pytest.raises(type(e)):
                decode_png(data, cuda_device)
            continue
        assert np.array_equal(decode_png(data, cuda_device).cpu().numpy(), want), name


def test_two_decodes_are_identical(cuda_device, corpus):
    for name in ('smooth_RGB_4032x3024', 'photo_RGB_1023x769', 'zlib_fixed_RGB_200x150'):
        a, sa = _device_status(corpus[name], cuda_device)
        b, sb = _device_status(corpus[name], cuda_device)
        assert sa == sb == 0 and torch.equal(a, b), name


def test_truncated_streams_report_status(cuda_device, corpus):
    from dust3r_b200.utils.image import _png_launch, _png_stage
    for name in ('pil_RGB_53x37', 'photo_RGB_1023x769', 'zlib_fixed_RGB_200x150'):
        desc, size, pinned = _png_stage(corpus[name])
        for cut in (6, int(pinned.numel()) // 2, int(pinned.numel()) - 1):
            desc.idat_bytes = cut
            _, status = _png_launch((desc, size, pinned[:cut].clone()), cuda_device)
            assert int(status.item()) != 0, (name, cut)


@pytest.fixture(scope='module')
def mixed_folder(tmp_path_factory):
    d = tmp_path_factory.mktemp('mixed_png')
    (d / 'a_baseline.jpg').write_bytes(_pil_jpeg(_pixels(300, 400, 31), quality=90, subsampling=2))
    (d / 'b_progressive.jpg').write_bytes(_pil_jpeg(_pixels(300, 400, 32), quality=90, progressive=True))
    (d / 'c_rgb.png').write_bytes(pil_png(pixels(240, 320, 33, 'photo'), 'RGB'))
    (d / 'd_grey.png').write_bytes(pil_png(pixels(320, 256, 34, 'photo', 1), 'L'))
    (d / 'e_rgba.PNG').write_bytes(pil_png(pixels(200, 280, 35, 'photo', 4), 'RGBA'))
    idx = pixels(250, 300, 36, 'noise', 1) % 40
    pal = np.random.default_rng(37).integers(0, 256, (40, 3), dtype=np.uint8)
    (d / 'f_palette.png').write_bytes(raw_png(idx, 3, palette=pal))
    (d / 'g_rotated.png').write_bytes(raw_png(pixels(240, 320, 38, 'photo'), 2, before=[(b'eXIf', exif_bytes(6))]))
    (d / 'h_refused.png').write_bytes(crafted_streams()['long'][0])        # the kernels refuse it, Pillow decodes it
    (d / 'i_4bit.png').write_bytes(excluded_files()['palette_4bit'][0])   # sent to Pillow by its header
    (d / 'j_notes.txt').write_text('skipped')
    return str(d)


@pytest.fixture
def every_png_on_device(monkeypatch):
    """load_images routes PNGs of any size to the GPU decoder (by default only those of PNG_DEVICE_MIN_PIXELS or more)."""
    from dust3r_b200.utils import image
    monkeypatch.setattr(image, 'PNG_DEVICE_MIN_PIXELS', 0)


@pytest.mark.parametrize('workers', [1, 3, 4])
def test_load_images_device_equals_host(cuda_device, mixed_folder, workers, every_png_on_device):
    import os
    from dust3r_b200.utils.image import _device_stage
    host, host_log = _load(mixed_folder, None, workers)
    dev, dev_log = _load(mixed_folder, cuda_device, workers)
    assert dev_log == host_log and len(host) == 9
    for h, d in zip(host, dev):
        assert d['img'].device.type == 'cuda'
        assert torch.equal(d['img'].cpu(), h['img']), h['idx']
        assert np.array_equal(d['true_shape'], h['true_shape']) and d['idx'] == h['idx'] and d['instance'] == h['instance']
    on_device = [n for n in sorted(os.listdir(mixed_folder)) if n.lower().endswith('.png')
                 and _device_stage(open(os.path.join(mixed_folder, n), 'rb').read()) is not None]
    assert len(on_device) == 6                                # every PNG but the 4-bit one takes the device path


def test_load_images_routes_large_pngs_by_default(cuda_device, corpus, tmp_path):
    """With the default threshold the 4032x3024 file is decoded on the GPU and a small one by Pillow; both equal the host path."""
    from dust3r_b200.utils.image import _device_stage
    (tmp_path / 'a_large.png').write_bytes(corpus['smooth_RGB_4032x3024'])
    (tmp_path / 'b_small.png').write_bytes(corpus['pil_RGB_53x37'])
    assert _device_stage(corpus['smooth_RGB_4032x3024']) is not None and _device_stage(corpus['pil_RGB_53x37']) is None
    host, host_log = _load(str(tmp_path), None, 2)
    dev, dev_log = _load(str(tmp_path), cuda_device, 2)
    assert dev_log == host_log
    for h, d in zip(host, dev):
        assert torch.equal(d['img'].cpu(), h['img']), h['idx']


def test_inference_on_png_loaded_views_equals_host_loaded(cuda_device, mixed_folder, every_png_on_device):
    from dust3r_b200.config import ModelConfig
    from dust3r_b200.image_pairs import make_pairs
    from dust3r_b200.inference import inference
    from dust3r_b200.model import AsymmetricCroCo3DStereo
    from dust3r_b200.utils.synth import synth_state_dict
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
