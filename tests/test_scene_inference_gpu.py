"""Encode once, decode by index: model.encode_images / model.decode_pairs (d3r_encode_images / d3r_decode_pairs) and the
inference() paths built on them, against the paths that existed before them.

Every comparison is bit for bit: each kernel computes an image (or a token row) independently of the rest of its launch, so
encoding an image once and decoding its pairs in any batch gives the bits of forward() on that pair."""
import ctypes as C

import numpy as np
import pytest
import torch

from dust3r_b200 import _lib
from dust3r_b200.image_pairs import make_pairs
from dust3r_b200.utils.device import collate_with_cat, to_cpu
from dust3r_b200.utils.synth import synth_images

pytestmark = pytest.mark.gpu

KEYS = (('pred1', 'pts3d'), ('pred1', 'conf'), ('pred2', 'pts3d_in_other_view'), ('pred2', 'conf'))


def _small_cfgs():
    from test_oracle import _small_cfgs as f
    return f()


def _net(cfg, device, seed=11):
    from test_forward_gpu import _build
    assert not cfg.landscape_only    # the small configs and the published ones are built with landscape_only=False
    net, sd = _build(cfg, seed, device)
    return net, sd


def _images(sizes, seed):
    out = []
    for k, (h, w) in enumerate(sizes):
        v = synth_images(1, h, w, seed=seed + k)[0]
        out.append(dict(v, idx=k, instance=str(k)))
    return out


def _assert_same(a, b, path='out'):
    """Same structure (types, keys and their order, lengths), same values, bit for bit."""
    assert type(a) is type(b), (path, type(a), type(b))
    if isinstance(a, dict):
        assert list(a) == list(b), (path, list(a), list(b))
        for k in a:
            _assert_same(a[k], b[k], f'{path}.{k}')
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), (path, len(a), len(b))
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, f'{path}[{i}]')
    elif torch.is_tensor(a):
        assert a.dtype == b.dtype and a.shape == b.shape and a.device == b.device, (path, a.dtype, b.dtype, a.shape, b.shape)
        assert torch.equal(a, b), (path, float((a.float() - b.float()).abs().max()))
    else:
        assert a == b, (path, a, b)


def _patch_embed_rows(records, E):
    """Summed M of the patch-embedding GEMM launches (K = 3 * 16 * 16, N = enc_dim, plain GEMM)."""
    import re
    rows = 0
    for r in records:
        m = re.fullmatch(r'M=(\d+) N=(\d+) K=(\d+) flags=0x([0-9a-f]+) mode=(\d+) epi=(\d+)', r['detail'])
        if r['tag'].startswith('gemm_') and m and int(m.group(3)) == 768 and int(m.group(2)) == E and m.group(5) == '0':
            rows += int(m.group(1))
    return rows


# ---- same-size scenes ----------------------------------------------------------------------------------------------------
@pytest.mark.timeout(1200)
@pytest.mark.parametrize('name', ['small_dpt', 'small_linear'])
def test_same_size_scene_equals_private_copies(cuda_device, name):
    """A make_pairs list shares one image dict between many pairs: inference() encodes every image once and decodes each
    micro-batch from those features.  The same list with private copies of every image takes the all-distinct path
    (both images of every pair encoded in the batch): the two must agree bit for bit, for every graph and batch size."""
    from dust3r_b200.inference import inference
    cfg, H, W = _small_cfgs()[name]
    net, _ = _net(cfg, cuda_device)
    imgs = _images([(H, W)] * 6, seed=30)
    for graph, sym in (('complete', True), ('complete', False), ('swin-2', True), ('oneref-2', True)):
        pairs = make_pairs(imgs, scene_graph=graph, prefilter=None, symmetrize=sym)
        private = [(dict(a, img=a['img'].clone()), dict(b, img=b['img'].clone())) for a, b in pairs]
        for bs in (1, 4, 16):
            a = inference(pairs, net, cuda_device, batch_size=bs, verbose=False)
            c = inference(private, net, cuda_device, batch_size=bs, verbose=False)
            for which, key in KEYS:
                assert torch.equal(a[which][key], c[which][key]), (graph, sym, bs, which, key)
            assert torch.equal(a['view1']['img'], c['view1']['img']) and a['view2']['idx'] == c['view2']['idx']


@pytest.mark.timeout(900)
def test_each_image_is_encoded_once(cuda_device):
    """Under the profiler, the patch-embedding GEMM launches of one inference() call over a shared-image scene add up to one
    encoder pass per distinct image (before, every micro-batch re-encoded the images it touched)."""
    from dust3r_b200.inference import inference
    cfg, H, W = _small_cfgs()['small_dpt']
    net, _ = _net(cfg, cuda_device)
    n = 7
    pairs = make_pairs(_images([(H, W)] * n, seed=40), scene_graph='complete', prefilter=None, symmetrize=True)
    inference(pairs[:2], net, cuda_device, batch_size=4, verbose=False)   # repack outside the profiled call
    torch.cuda.synchronize()
    _lib.prof_enable(True)
    try:
        inference(pairs, net, cuda_device, batch_size=4, verbose=False)
        torch.cuda.synchronize()
        recs = _lib.prof_dump()
    finally:
        _lib.prof_enable(False)
    assert _patch_embed_rows(recs, cfg.enc_embed_dim) == n * (H // 16) * (W // 16)


# ---- mixed sizes ---------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(1500)
@pytest.mark.parametrize('name', ['small_dpt', 'small_linear'])
def test_mixed_sizes_equal_the_per_pair_loop(cuda_device, name):
    """Three sizes plus a landscape / portrait mix (H x W and W x H) and one size twice: inference() groups the pairs by
    (size of view 1, size of view 2) and decodes each group in batches.  It must return what the one-pair-per-call loop
    returned before, element by element and bit for bit, with the same structure, at every batch size and option."""
    from dust3r_b200.inference import inference, loss_of_one_batch
    cfg, H, W = _small_cfgs()[name]
    net, _ = _net(cfg, cuda_device)
    sizes = [(H, W), (W, H), (H - 16, W), (H, W - 32), (H, W)]
    pairs = make_pairs(_images(sizes, seed=50), scene_graph='complete', prefilter=None, symmetrize=True)
    ref = collate_with_cat([to_cpu(loss_of_one_batch(collate_with_cat([p]), net, None, cuda_device)) for p in pairs], lists=True)
    ref_noimg = dict(ref, view1={k: v for k, v in ref['view1'].items() if k != 'img'},
                     view2={k: v for k, v in ref['view2'].items() if k != 'img'})
    for bs in (1, 4, 16):
        _assert_same(inference(pairs, net, cuda_device, batch_size=bs, verbose=False), ref)
    for kw in (dict(keep_on_device=True), dict(return_images=False), dict(keep_on_device=True, return_images=False)):
        out = inference(pairs, net, cuda_device, batch_size=4, verbose=False, **kw)
        if kw.get('keep_on_device'):
            assert out['pred1']['pts3d'][0].is_cuda
            assert not kw.get('return_images', True) or out['view1']['img'][0].is_cuda
        _assert_same(to_cpu(out), ref if kw.get('return_images', True) else ref_noimg)


# ---- the public API ------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_encode_images_is_the_forward_encoder_output(cuda_device):
    """encode_images == debug tap 4 (enc_norm output) of the packed model's forward, bit for bit, and the oracle's enc_norm
    stage within the stage tolerance."""
    from oracle.forward_oracle import forward_oracle
    cfg, H, W = _small_cfgs()['small_dpt']
    net, sd = _net(cfg, cuda_device)
    imgs = synth_images(4, H, W, seed=7)
    img1 = torch.cat([imgs[0]['img'], imgs[2]['img']])
    img2 = torch.cat([imgs[1]['img'], imgs[3]['img']])
    st = {}
    forward_oracle(sd, cfg, img1, img2, ['0', '2'], ['1', '3'], stages=st)
    x = torch.cat((img1, img2)).to(cuda_device)
    feat = net.encode_images(x)
    N, E = (H // 16) * (W // 16), cfg.enc_embed_dim
    assert feat.dtype == torch.bfloat16 and feat.shape == (4, H // 16, W // 16, E) and feat.is_cuda
    packed = net._packed
    idx1, idx2 = np.arange(2, dtype=np.int32), 2 + np.arange(2, dtype=np.int32)
    tap = torch.zeros((4 * N * E,), dtype=torch.float32, device=cuda_device)
    packed.forward(x, idx1, idx2, 2, H, W, debug=(4, tap))
    torch.cuda.synchronize()
    assert torch.equal(feat.float().reshape(-1), tap)
    ref = st['enc_norm'].reshape(-1)
    assert float((feat.float().cpu().reshape(-1) - ref).norm() / ref.norm()) < 2e-2


@pytest.mark.timeout(900)
@pytest.mark.parametrize('name', ['small_dpt', 'small_linear'])
def test_add_a_view_to_a_scene(cuda_device, name):
    """Encode k images, later encode image k alone and decode only the pairs it adds, from the two feature sets: the result
    equals inference() on the whole (k + 1)-view list, bit for bit."""
    from dust3r_b200.inference import inference
    cfg, H, W = _small_cfgs()[name]
    net, _ = _net(cfg, cuda_device)
    k = 5
    imgs = _images([(H, W)] * (k + 1), seed=60)
    old = net.encode_images(torch.cat([v['img'] for v in imgs[:k]]).to(cuda_device))
    new = net.encode_images(imgs[k]['img'].to(cuda_device))
    pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=True)
    whole = inference(pairs, net, cuda_device, batch_size=4, verbose=False)
    rows_a = [i for i, (a, b) in enumerate(pairs) if b['idx'] == k]    # (old view, new view)
    rows_b = [i for i, (a, b) in enumerate(pairs) if a['idx'] == k]    # (new view, old view)
    assert len(rows_a) == len(rows_b) == k
    ra = net.decode_pairs(old, [pairs[i][0]['idx'] for i in rows_a], new, [0] * k)
    rb = net.decode_pairs(new, [0] * k, old, [pairs[i][1]['idx'] for i in rows_b])
    for rows, (r1, r2) in ((rows_a, ra), (rows_b, rb)):
        for which, key in KEYS:
            got = (r1 if which == 'pred1' else r2)[key].cpu()
            assert torch.equal(got, whole[which][key][rows]), (which, key)


@pytest.mark.timeout(900)
def test_decode_two_sizes_equals_forward(cuda_device):
    """decode_pairs over a landscape and a portrait feature set == model.forward() on the same pairs (two-size batch)."""
    cfg, H, W = _small_cfgs()['small_dpt']
    net, _ = _net(cfg, cuda_device)
    a = torch.cat([v['img'] for v in synth_images(3, H, W, seed=70)]).to(cuda_device)
    b = torch.cat([v['img'] for v in synth_images(2, W, H, seed=80)]).to(cuda_device)
    fa, fb = net.encode_images(a), net.encode_images(b)
    i1, i2 = [2, 0, 1, 2], [1, 1, 0, 0]
    r1, r2 = net.decode_pairs(fa, i1, fb, i2)
    q1, q2 = net(dict(img=a[i1], instance=['a'] * 4), dict(img=b[i2], instance=['b'] * 4))
    _assert_same(r1, q1)
    _assert_same(r2, q2)
    assert r1['pts3d'].shape == (4, H, W, 3) and r2['pts3d_in_other_view'].shape == (4, W, H, 3)


@pytest.mark.timeout(600)
def test_rejected_arguments_launch_nothing(cuda_device):
    """Wrong indices, dtypes, shapes, devices, sizes and alignments are argument errors, raised before any launch."""
    from dust3r_b200._lib import D3RError
    cfg, H, W = _small_cfgs()['small_linear']
    net, _ = _net(cfg, cuda_device)
    x = torch.cat([v['img'] for v in synth_images(3, H, W, seed=90)]).to(cuda_device)
    feat = net.encode_images(x)
    torch.cuda.synchronize()
    packed, lib = net._packed, net._packed.lib
    before = _lib.launch_count()
    bad_py = [
        lambda: net.decode_pairs(feat, [0, 3], feat, [1, 2]),                        # index out of range
        lambda: net.decode_pairs(feat, [-1], feat, [0]),
        lambda: net.decode_pairs(feat.float(), [0], feat, [1]),                      # wrong dtype
        lambda: net.decode_pairs(feat[..., :64].contiguous(), [0], feat, [1]),       # wrong feature width
        lambda: net.decode_pairs(feat[0], [0], feat, [1]),                           # wrong rank
        lambda: net.decode_pairs(feat.cpu(), [0], feat, [1]),                        # wrong device
        lambda: net.decode_pairs(feat, [0, 1], feat, [1]),                           # index lists of two lengths
        lambda: net.decode_pairs(feat, [0.0], feat, [1.0]),
        lambda: net.encode_images(x[:, :2]),
    ]
    for call in bad_py:
        with pytest.raises(ValueError):
            call()
    with pytest.raises(D3RError):
        net.encode_images(x.cpu())
    assert _lib.launch_count() == before
    # the C entry points check by themselves (the features come from outside the library)
    m = C.byref(packed.cmodel)
    ws = torch.empty((max(lib.d3r_decode_workspace_bytes(m, 2, H, W, H, W), lib.d3r_encode_workspace_bytes(m, 3, H, W)),),
                     dtype=torch.uint8, device=cuda_device)
    out = [torch.empty((2, H, W, 3), device=cuda_device) for _ in range(2)]
    conf = [torch.empty((2, H, W), device=cuda_device) for _ in range(2)]
    st = _lib.stream_ptr()

    def dec(f1, n1, h1, w1, f2, n2, h2, w2, i1, i2):
        a, b = (C.c_int32 * 2)(*i1), (C.c_int32 * 2)(*i2)
        return lib.d3r_decode_pairs(m, f1, n1, h1, w1, f2, n2, h2, w2, a, b, 2, out[0].data_ptr(), conf[0].data_ptr(),
                                    out[1].data_ptr(), conf[1].data_ptr(), ws.data_ptr(), ws.numel(), st)

    p = feat.data_ptr()
    assert dec(p, 3, H, W, p, 3, H, W, [0, 1], [2, 1]) == 0                    # the valid call, checked below for no launch
    torch.cuda.synchronize()
    before = _lib.launch_count()
    rcs = [dec(p, 3, H, W, p, 3, H, W, [0, 3], [1, 2]),                       # index out of range
           dec(p, 3, H, W, p, 3, H, W - 16, [0, 1], [1, 2]),                  # one buffer described with two sizes
           dec(p + 2, 3, H, W, p, 3, H, W, [0, 1], [1, 2]),                   # misaligned features
           dec(p, 3, H, W + 8, p, 3, H, W, [0, 1], [1, 2]),                   # not a multiple of the patch
           dec(None, 3, H, W, p, 3, H, W, [0, 1], [1, 2]),                    # null features
           dec(p, 0, H, W, p, 3, H, W, [0, 1], [1, 2]),                       # empty feature set
           lib.d3r_encode_images(m, x.data_ptr(), 3, H, W, p + 2, ws.data_ptr(), ws.numel(), st),
           lib.d3r_encode_images(m, x.data_ptr(), 3, H, W, p, ws.data_ptr(), 1024, st)]       # workspace too small
    assert all(rc != 0 for rc in rcs), rcs
    assert _lib.launch_count() == before
    assert lib.d3r_encode_workspace_bytes(m, 0, H, W) < 0 and lib.d3r_decode_workspace_bytes(m, 0, H, W, H, W) < 0


@pytest.mark.timeout(600)
@pytest.mark.parametrize('name', ['small_dpt', 'small_linear'])
def test_calls_write_only_inside_their_buffers(cuda_device, name):
    """An encode call writes nothing past the workspace size its query returns or past the features, and a decode call
    nothing past its workspace: sentinel bytes behind each buffer stay as they were.  The small DPT model's encoder is
    narrower than a patch (4 x 128 < 3 x 16 x 16), so its patch im2col is wider than its MLP hidden layer."""
    cfg, H, W = _small_cfgs()[name]
    net, _ = _net(cfg, cuda_device)
    x = torch.cat([v['img'] for v in synth_images(3, H, W, seed=95)]).to(cuda_device)
    packed, lib = net.repack(), net._packed.lib
    m, st, tail = C.byref(packed.cmodel), _lib.stream_ptr(), 1 << 20
    n_feat = 3 * (H // 16) * (W // 16) * cfg.enc_embed_dim * 2
    need_e, need_d = lib.d3r_encode_workspace_bytes(m, 3, H, W), lib.d3r_decode_workspace_bytes(m, 2, H, W, H, W)
    ws_e, feat, ws_d = [torch.full((n + tail,), 0xA5, dtype=torch.uint8, device=cuda_device) for n in (need_e, n_feat, need_d)]
    out = [torch.empty((2, H, W, 3), device=cuda_device) for _ in range(2)]
    conf = [torch.empty((2, H, W), device=cuda_device) for _ in range(2)]
    assert lib.d3r_encode_images(m, x.data_ptr(), 3, H, W, feat.data_ptr(), ws_e.data_ptr(), need_e, st) == 0
    i1, i2 = (C.c_int32 * 2)(0, 1), (C.c_int32 * 2)(2, 0)
    assert lib.d3r_decode_pairs(m, feat.data_ptr(), 3, H, W, feat.data_ptr(), 3, H, W, i1, i2, 2, out[0].data_ptr(),
                                conf[0].data_ptr(), out[1].data_ptr(), conf[1].data_ptr(), ws_d.data_ptr(), need_d, st) == 0
    torch.cuda.synchronize()
    for what, buf, n in (('encode workspace', ws_e, need_e), ('features', feat, n_feat), ('decode workspace', ws_d, need_d)):
        assert bool((buf[n:] == 0xA5).all()), what
    ref = net.encode_images(x)
    assert torch.equal(feat[:n_feat].view(torch.bfloat16).reshape(ref.shape), ref)


# ---- the published model -------------------------------------------------------------------------------------------------
@pytest.mark.timeout(1800)
def test_published_vitl_512_dpt_scene(cuda_device):
    """vitl_512_dpt at 512x384: a shared-image scene equals private copies, and a landscape / portrait scene equals the
    per-pair loop, bit for bit; each distinct image is encoded once in both."""
    from dust3r_b200.config import vitl_512_dpt
    from dust3r_b200.inference import inference, loss_of_one_batch
    cfg, H, W = vitl_512_dpt(), 384, 512
    net, _ = _net(cfg, cuda_device, seed=0)
    imgs = _images([(H, W)] * 4, seed=100)
    pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=True)
    private = [(dict(a, img=a['img'].clone()), dict(b, img=b['img'].clone())) for a, b in pairs]
    c = inference(private, net, cuda_device, batch_size=8, verbose=False)
    torch.cuda.synchronize()
    _lib.prof_enable(True)
    try:
        a = inference(pairs, net, cuda_device, batch_size=8, verbose=False)
        torch.cuda.synchronize()
        recs = _lib.prof_dump()
    finally:
        _lib.prof_enable(False)
    assert _patch_embed_rows(recs, cfg.enc_embed_dim) == 4 * (H // 16) * (W // 16)
    for which, key in KEYS:
        assert torch.equal(a[which][key], c[which][key]), (which, key)
    mixed = _images([(H, W), (W, H), (H, W)], seed=110)
    pairs = make_pairs(mixed, scene_graph='complete', prefilter=None, symmetrize=True)
    ref = collate_with_cat([to_cpu(loss_of_one_batch(collate_with_cat([p]), net, None, cuda_device)) for p in pairs], lists=True)
    _assert_same(inference(pairs, net, cuda_device, batch_size=4, verbose=False), ref)
