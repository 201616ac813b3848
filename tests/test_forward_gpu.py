"""Pairwise forward on the H100 path vs the CPU fp32 oracle / the reference's golden outputs.

Numerics: GEMM operands are bf16 (8-bit mantissa), accumulation and the residual stream are fp32; the
reference computes in fp32 (TF32 on GPU).  Stated tolerances (calibrated on the synthetic-weight models):
  * pre-postprocess head output (log-space):  |err| <= 0.06 absolute  (values are O(1))
  * pts3d:  rel. L2 error per image <= 3e-2, conf: rel. L2 <= 3e-2
Pair ordering / indexing is compared exactly."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from dust3r_b200.utils.synth import synth_state_dict, synth_images
from dust3r_b200.image_pairs import make_pairs

pytestmark = pytest.mark.gpu


def _small_cfgs():
    from test_oracle import _small_cfgs as f
    return f()


def _build(cfg, seed, device):
    from dust3r_b200.model import AsymmetricCroCo3DStereo
    net = AsymmetricCroCo3DStereo(pos_embed=cfg.pos_embed, img_size=cfg.img_size, head_type=cfg.head_type,
                                  depth_mode=cfg.depth_mode, conf_mode=cfg.conf_mode, enc_embed_dim=cfg.enc_embed_dim,
                                  enc_depth=cfg.enc_depth, enc_num_heads=cfg.enc_num_heads, dec_embed_dim=cfg.dec_embed_dim,
                                  dec_depth=cfg.dec_depth, dec_num_heads=cfg.dec_num_heads, landscape_only=cfg.landscape_only)
    sd = synth_state_dict(cfg, seed=seed)
    net.load_state_dict(sd, strict=True)
    return net.to(device), sd


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-12))


@pytest.mark.timeout(600)
@pytest.mark.parametrize('impl', [2, 3])
def test_attention_matches_torch(cuda_device, impl):
    from dust3r_b200 import _lib
    lib = _lib.get_lib()
    lib.d3r_set_attention_impl(impl)
    g = torch.Generator().manual_seed(0)
    # the last two shapes give the persistent kernel (impl 2) several tiles per CTA, one of them with ragged key blocks
    for (B, Hh, Nq, Nk) in [(2, 3, 24, 24), (1, 2, 196, 196), (2, 4, 768, 768), (1, 2, 100, 37), (3, 1, 65, 130),
                            (6, 16, 768, 768), (40, 8, 100, 137)]:
        q = torch.randn((B, Nq, Hh, 64), generator=g).to(cuda_device).bfloat16()
        k = torch.randn((B, Nk, Hh, 64), generator=g).to(cuda_device).bfloat16()
        v = torch.randn((B, Nk, Hh, 64), generator=g).to(cuda_device).bfloat16()
        out = torch.full((B, Nq, Hh, 64), float('nan'), dtype=torch.bfloat16, device=cuda_device)
        ld = Hh * 64
        _lib.check(lib.d3r_attention_hd64(q.data_ptr(), ld, k.data_ptr(), ld, v.data_ptr(), ld, out.data_ptr(), ld,
                                          B, Hh, Nq, Nk, 0.125, _lib.stream_ptr()))
        torch.cuda.synchronize()
        qf, kf, vf = [t.float().permute(0, 2, 1, 3) for t in (q, k, v)]
        ref = (torch.softmax(qf @ kf.transpose(-1, -2) * 0.125, dim=-1) @ vf).permute(0, 2, 1, 3)
        assert torch.isfinite(out.float()).all()
        err = (out.float() - ref).abs().max().item()
        lib.d3r_set_attention_impl(3) if err >= 2e-2 else None
        assert err < 2e-2, (impl, B, Hh, Nq, Nk, err)
    lib.d3r_set_attention_impl(3)


@pytest.mark.timeout(600)
@pytest.mark.parametrize('impl', [2, 3])
def test_attention_growing_scores_move_the_reference(cuda_device, impl):
    """Keys whose logits grow along the sequence (by far more than the 2^8 headroom of the lazy exponent reference) force the
    online softmax to move its reference and rescale O / l several times per row; masked (ragged) last block included."""
    from dust3r_b200 import _lib
    lib = _lib.get_lib()
    lib.d3r_set_attention_impl(impl)
    g = torch.Generator().manual_seed(1)
    try:
        for (B, Hh, Nq, Nk) in [(2, 2, 256, 768), (1, 3, 130, 700)]:
            q = torch.randn((B, Nq, Hh, 64), generator=g)
            k = torch.randn((B, Nk, Hh, 64), generator=g)
            # logits of key n ~ q.k * (1 + 9 n / Nk) + a rising offset along q's own direction
            ramp = torch.linspace(1.0, 10.0, Nk).view(1, Nk, 1, 1)
            k = k * ramp + 0.35 * ramp * q.mean(dim=1, keepdim=True)
            v = torch.randn((B, Nk, Hh, 64), generator=g)
            q, k, v = [t.to(cuda_device).bfloat16() for t in (q, k, v)]
            out = torch.full((B, Nq, Hh, 64), float('nan'), dtype=torch.bfloat16, device=cuda_device)
            ld = Hh * 64
            _lib.check(lib.d3r_attention_hd64(q.data_ptr(), ld, k.data_ptr(), ld, v.data_ptr(), ld, out.data_ptr(), ld,
                                              B, Hh, Nq, Nk, 0.125, _lib.stream_ptr()))
            torch.cuda.synchronize()
            qf, kf, vf = [t.float().permute(0, 2, 1, 3) for t in (q, k, v)]
            logits = qf @ kf.transpose(-1, -2) * 0.125
            # the scenario is only meaningful if row maxima really outgrow the first block's by more than the headroom
            growth = (logits.max(dim=-1).values - logits[..., :128].max(dim=-1).values) * 1.4427
            assert float(growth.max()) > 16
            ref = (torch.softmax(logits, dim=-1) @ vf).permute(0, 2, 1, 3)
            assert torch.isfinite(out.float()).all()
            err = (out.float() - ref).abs().max().item()
            assert err < 3e-2, (impl, B, Hh, Nq, Nk, err)
    finally:
        lib.d3r_set_attention_impl(3)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('name', ['small_linear', 'small_dpt'])
def test_forward_matches_oracle_and_reference_golden(cuda_device, name):
    from dust3r_b200.inference import inference
    from oracle.forward_oracle import forward_oracle
    cfg, H, W = _small_cfgs()[name]
    net, sd = _build(cfg, 11, cuda_device)
    imgs = synth_images(3, H, W, seed=5)
    pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=True)
    out = inference(pairs, net, cuda_device, batch_size=4, verbose=False)
    gold = np.load(os.path.join(GOLDEN, f'forward_{name}.npz'))
    # bit-exact pair indexing
    assert out['view1']['idx'] == gold['idx1'].tolist() and out['view2']['idx'] == gold['idx2'].tolist()
    assert all(t.device.type == 'cpu' for t in (out['pred1']['pts3d'], out['pred2']['conf']))
    for got, key in ((out['pred1']['pts3d'], 'pts3d'), (out['pred1']['conf'], 'conf1'),
                     (out['pred2']['pts3d_in_other_view'], 'pts3d_in_other_view'), (out['pred2']['conf'], 'conf2')):
        ref = torch.from_numpy(gold[key])
        assert got.shape == ref.shape and torch.isfinite(got).all()
        for b in range(ref.shape[0]):
            assert _rel(got[b], ref[b]) < 3e-2, (key, b, _rel(got[b], ref[b]))


@pytest.mark.timeout(900)
@pytest.mark.parametrize('name', ['small_dpt', 'small_linear'])
def test_forward_mixed_sizes_matches_reference_golden(cuda_device, name):
    """Three images of three sizes, all ordered pairs: inference() returns lists (inference.py:60-72) and every pair
    runs through one encode call per size and d3r_decode_pairs (cross-attention between two token grids)."""
    from dust3r_b200.inference import inference
    cfg, H, W = _small_cfgs()[name]
    net, sd = _build(cfg, 11, cuda_device)
    sizes = [(H, W), (H - 16, W), (H, W - 32)]
    imgs = [dict(synth_images(1, h, w, seed=20 + k)[0], idx=k, instance=str(k)) for k, (h, w) in enumerate(sizes)]
    pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=True)
    out = inference(pairs, net, cuda_device, batch_size=4, verbose=False)
    gold = np.load(os.path.join(GOLDEN, f'forward_{name}_mixed.npz'))
    assert out['view1']['idx'] == gold['idx1'].tolist() and out['view2']['idx'] == gold['idx2'].tolist()
    assert isinstance(out['pred1']['pts3d'], list) and len(out['pred1']['pts3d']) == len(pairs)
    for k in range(len(pairs)):
        for got, key in ((out['pred1']['pts3d'][k], f'pts3d_{k}'), (out['pred1']['conf'][k], f'conf1_{k}'),
                         (out['pred2']['pts3d_in_other_view'][k], f'pts3d_in_other_view_{k}'), (out['pred2']['conf'][k], f'conf2_{k}')):
            ref = torch.from_numpy(gold[key])
            got = got.reshape(ref.shape) if got.numel() == ref.numel() else got
            assert got.shape == ref.shape and got.device.type == 'cpu' and torch.isfinite(got).all(), (key, got.shape, ref.shape)
            assert _rel(got, ref) < 3e-2, (key, _rel(got, ref))


@pytest.mark.timeout(900)
def test_inference_pipelined_micro_batches_bit_identical(cuda_device):
    """batch_size >= 16 runs as two pipelined halves (upload / compute / download overlap): the result must be
    bit-identical to small unpipelined batches, in pair order, for symmetrised and plain pair lists."""
    from dust3r_b200.inference import inference, _micro_batch
    assert _micro_batch(8) == 8 and _micro_batch(16) == 8 and _micro_batch(32) == 16 and _micro_batch(18) == 10
    cfg, H, W = _small_cfgs()['small_dpt']
    net, sd = _build(cfg, 11, cuda_device)
    imgs = synth_images(5, H, W, seed=9)
    for sym in (True, False):
        pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=sym)
        a = inference(pairs, net, cuda_device, batch_size=4, verbose=False)
        b = inference(pairs, net, cuda_device, batch_size=16, verbose=False)
        assert a['view1']['idx'] == b['view1']['idx'] and a['view2']['idx'] == b['view2']['idx']
        assert torch.equal(a['view1']['img'], b['view1']['img']) and torch.equal(a['view2']['img'], torch.cat([p[1]['img'] for p in pairs]))
        for which, key in (('pred1', 'pts3d'), ('pred1', 'conf'), ('pred2', 'pts3d_in_other_view'), ('pred2', 'conf')):
            assert torch.equal(a[which][key], b[which][key]), (sym, which, key)
        # make_pairs shares one image dict between many pairs -> inference() encodes each distinct image once per
        # batch (index maps).  With private copies of every image it falls back to encoding both images of every
        # pair, like the reference: the two must agree bit for bit.
        private = [(dict(x, img=x['img'].clone()), dict(y, img=y['img'].clone())) for x, y in pairs]
        c = inference(private, net, cuda_device, batch_size=16, verbose=False)
        for which, key in (('pred1', 'pts3d'), ('pred1', 'conf'), ('pred2', 'pts3d_in_other_view'), ('pred2', 'conf')):
            assert torch.equal(a[which][key], c[which][key]), ('private copies', sym, which, key)
        assert torch.equal(a['view1']['img'], c['view1']['img'])


@pytest.mark.timeout(900)
def test_forward_stages_against_oracle(cuda_device):
    """Stage taps of the forward vs the oracle's intermediate tensors (small DPT model, 2 pairs)."""
    from oracle.forward_oracle import forward_oracle
    cfg, H, W = _small_cfgs()['small_dpt']
    net, sd = _build(cfg, 11, cuda_device)
    imgs = synth_images(4, H, W, seed=7)
    img1 = torch.cat([imgs[0]['img'], imgs[2]['img']])
    img2 = torch.cat([imgs[1]['img'], imgs[3]['img']])
    st = {}
    o1, o2 = forward_oracle(sd, cfg, img1, img2, ['0', '2'], ['1', '3'], stages=st)
    packed = net.repack()
    N = (H // 16) * (W // 16)
    E, D = cfg.enc_embed_dim, cfg.dec_embed_dim
    taps = {1: ('patch_embed', 4 * N * E), 2: ('enc_block0', 4 * N * E), 3: (f'enc_block{cfg.enc_depth - 1}', 4 * N * E),
            4: ('enc_norm', 4 * N * E), 5: ('decoder_embed1', 2 * N * D), 6: ('dec_block0_1', 2 * N * D),
            7: ('dec_block0_2', 2 * N * D), 8: (f'dec_block{cfg.dec_depth - 1}_1', 2 * N * D)}
    imgs_cat = torch.cat((img1, img2)).to(cuda_device)
    idx1, idx2 = np.arange(2, dtype=np.int32), 2 + np.arange(2, dtype=np.int32)
    for stage, (name, n) in taps.items():
        buf = torch.zeros((n,), dtype=torch.float32, device=cuda_device)
        r1, r2 = packed.forward(imgs_cat, idx1, idx2, 2, H, W, debug=(stage, buf))
        torch.cuda.synchronize()
        ref = st[name].reshape(-1)
        err = _rel(buf.cpu(), ref)
        assert err < 2e-2, (name, err)
    # head taps (bf16 NHWC) vs oracle NCHW
    for stage, name in ((20, 'dpt1_layer0'), (23, 'dpt1_layer3'), (24, 'dpt1_path4'), (21, 'dpt1_path1')):
        ref = st[name].permute(0, 2, 3, 1).contiguous()
        buf = torch.zeros((ref.numel(),), dtype=torch.float32, device=cuda_device)
        packed.forward(imgs_cat, idx1, idx2, 2, H, W, debug=(stage, buf))
        torch.cuda.synchronize()
        # the tap is overwritten by head 2 as well (same scratch); head 1 runs first, head 2 second -> compare to head 2
        ref2 = st[name.replace('dpt1', 'dpt2')].permute(0, 2, 3, 1).contiguous()
        err = min(_rel(buf.cpu(), ref.reshape(-1)), _rel(buf.cpu(), ref2.reshape(-1)))
        assert err < 3e-2, (name, err)
    assert _rel(r1['pts3d'].cpu(), o1['pts3d']) < 3e-2
    assert _rel(r2['pts3d'].cpu(), o2['pts3d_in_other_view']) < 3e-2
    assert _rel(r1['conf'].cpu(), o1['conf']) < 3e-2


@pytest.mark.timeout(900)
def test_symmetrized_batch_uses_half_encoder_and_matches(cuda_device):
    """[(a,b),(b,a)] batches: the encoder only sees the even half (model.py:161-166); results must equal the
    unsymmetrised evaluation of the same pairs."""
    cfg, H, W = _small_cfgs()['small_linear']
    net, sd = _build(cfg, 11, cuda_device)
    imgs = synth_images(2, H, W, seed=8)
    a, b = imgs[0]['img'].to(cuda_device), imgs[1]['img'].to(cuda_device)
    v1 = dict(img=torch.cat((a, b)), instance=['0', '1'])
    v2 = dict(img=torch.cat((b, a)), instance=['1', '0'])
    r1, r2 = net(v1, v2)
    s1 = dict(img=torch.cat((a, b)), instance=['0', 'x'])   # breaks the symmetry test -> full encoder
    s2 = dict(img=torch.cat((b, a)), instance=['1', 'y'])
    q1, q2 = net(s1, s2)
    assert _rel(r1['pts3d'], q1['pts3d']) < 1e-5 and _rel(r2['pts3d_in_other_view'], q2['pts3d_in_other_view']) < 1e-5


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('name', ['vitl_224_linear', 'vitl_512_dpt'])
def test_published_architectures_match_reference_golden(cuda_device, name):
    """ViT-L/ViT-B at the published sizes vs strided samples of the unmodified reference's CPU output."""
    from dust3r_b200.config import vitl_224_linear, vitl_512_dpt
    from dust3r_b200.inference import inference
    cfg, H, W = (vitl_224_linear(), 224, 224) if name == 'vitl_224_linear' else (vitl_512_dpt(), 384, 512)
    net, sd = _build(cfg, 0, cuda_device)
    imgs = synth_images(2, H, W, seed=3)
    out = inference([(imgs[0], imgs[1])], net, cuda_device, batch_size=1, verbose=False)
    gold = np.load(os.path.join(GOLDEN, f'forward_{name}.npz'))
    s = int(gold['stride'])
    for got, key in ((out['pred1']['pts3d'], 'pts3d'), (out['pred1']['conf'], 'conf1'),
                     (out['pred2']['pts3d_in_other_view'], 'pts3d_in_other_view'), (out['pred2']['conf'], 'conf2')):
        ref = torch.from_numpy(gold[key])
        got = got[:, ::s, ::s]
        assert torch.isfinite(got).all()
        assert _rel(got, ref) < 4e-2, (key, _rel(got, ref))


@pytest.mark.timeout(1800)
def test_batched_forward_path_matches_oracle_and_error_is_operand_rounding(cuda_device):
    """The benchmark's code path: packed.forward on B = 16 distinct 512x384 pairs of the published ViT-L / ViT-B / DPT
    architecture (pair-GEMM policy, multi-tile persistent attention, M = 24576 / 49152 token GEMMs), compared per pair with the
    CPU oracle on three of the pairs (first, middle, last: a pair's result must not depend on its batch).

    Tolerance calibration (DESIGN.md section 2): the oracle is evaluated twice -- in the reference's fp32, and with every
    contraction's operands rounded to bf16 (fp32 accumulation), i.e. what any bf16-operand implementation computes.  The
    product must sit much closer to the second than the second sits to the first: the measured 1e-2 distance to the fp32
    reference is operand rounding, not implementation error."""
    import oracle.forward_oracle as fo
    from dust3r_b200.config import vitl_512_dpt
    cfg, H, W = vitl_512_dpt(), 384, 512
    net, sd = _build(cfg, 0, cuda_device)
    B = 16
    g = torch.Generator().manual_seed(77)
    imgs = torch.rand((2 * B, 3, H, W), generator=g) * 2 - 1
    packed = net.repack()
    idx1, idx2 = np.arange(B, dtype=np.int32), B + np.arange(B, dtype=np.int32)
    r1, r2 = packed.forward(imgs.to(cuda_device), idx1, idx2, B, H, W)
    torch.cuda.synchronize()
    assert torch.isfinite(r1['pts3d']).all() and torch.isfinite(r2['conf']).all()
    worst = dict(fp32=0.0, bf16=0.0, floor=0.0)
    for k in (0, B // 2, B - 1):
        a, b = imgs[k:k + 1], imgs[B + k:B + k + 1]
        o1, o2 = fo.forward_oracle(sd, cfg, a, b)
        with fo.operand_rounding(torch.bfloat16):
            e1, e2 = fo.forward_oracle(sd, cfg, a, b)
        for got, ref, emu in ((r1['pts3d'][k], o1['pts3d'][0], e1['pts3d'][0]), (r1['conf'][k], o1['conf'][0], e1['conf'][0]),
                              (r2['pts3d'][k], o2['pts3d_in_other_view'][0], e2['pts3d_in_other_view'][0]),
                              (r2['conf'][k], o2['conf'][0], e2['conf'][0])):
            got = got.cpu()
            worst['fp32'] = max(worst['fp32'], _rel(got, ref))
            worst['bf16'] = max(worst['bf16'], _rel(got, emu))
            worst['floor'] = max(worst['floor'], _rel(emu, ref))
        # per-pixel bound on the pointmap: 99.9 % of the pixels within 5 % of the scene scale (median point norm)
        d = (r1['pts3d'][k].cpu() - o1['pts3d'][0]).norm(dim=-1)
        scale = o1['pts3d'][0].norm(dim=-1).median()
        assert float(torch.quantile(d.flatten()[::7], 0.999)) < 0.05 * float(scale), (k, float(d.max()), float(scale))
    print('batched forward vs oracle: rel-L2 to fp32 oracle %.3e, to bf16-operand oracle %.3e; bf16-operand oracle vs fp32 oracle %.3e'
          % (worst['fp32'], worst['bf16'], worst['floor']))
    assert worst['fp32'] < 3e-2, worst
    assert worst['bf16'] < 0.6 * max(worst['floor'], 1e-3) + 2e-3, worst


@pytest.mark.timeout(900)
@pytest.mark.parametrize('name', ['small_linear', 'small_dpt'])
def test_landscape_only_many_ar_batch_matches_reference_golden(cuda_device, name):
    """landscape_only=True with transposed portrait items in the batch (ManyAR_PatchEmbed, patch_embed.py:42-70, and
    transpose_to_landscape.wrapper_yes, utils/misc.py:66-95): all four orientation combinations of a pair in one batch,
    against the output of the unmodified reference in that configuration."""
    import copy
    from dust3r_b200.utils.synth import many_ar_inputs
    cfg0, _, _ = _small_cfgs()[name]
    cfg = copy.deepcopy(cfg0)
    cfg.landscape_only = True
    net, sd = _build(cfg, 11, cuda_device)
    assert net.landscape_only
    gold = np.load(os.path.join(GOLDEN, f'forward_{name}_manyar.npz'))
    H, W = int(gold['H']), int(gold['W'])
    v1, v2 = many_ar_inputs(H, W)
    v1 = dict(v1, img=v1['img'].to(cuda_device))
    v2 = dict(v2, img=v2['img'].to(cuda_device))
    r1, r2 = net(v1, v2)
    for got, key in ((r1['pts3d'], 'pts3d'), (r1['conf'], 'conf1'), (r2['pts3d_in_other_view'], 'pts3d_in_other_view'), (r2['conf'], 'conf2')):
        ref = torch.from_numpy(gold[key])
        assert got.shape == ref.shape
        for k in range(4):
            assert _rel(got[k].cpu(), ref[k]) < 3e-2, (name, key, k, _rel(got[k].cpu(), ref[k]))


def test_in_place_weight_edit_is_picked_up(cuda_device):
    """The kernel-side operand buffers are rebuilt when a parameter was modified in place since the last packing."""
    cfg, H, W = _small_cfgs()['small_linear']
    net, sd = _build(cfg, 11, cuda_device)
    imgs = synth_images(2, H, W, seed=8)
    v1 = dict(img=imgs[0]['img'].to(cuda_device), instance=['0'])
    v2 = dict(img=imgs[1]['img'].to(cuda_device), instance=['1'])
    a, _ = net(v1, v2)
    a = a['pts3d'].clone()
    b, _ = net(v1, v2)
    assert torch.equal(a, b['pts3d'])
    with torch.no_grad():
        net.enc_norm.weight.mul_(1.5)
    c, _ = net(v1, v2)
    assert not torch.equal(a, c['pts3d'])


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('name', ['small_linear', 'small_dpt'])
@pytest.mark.parametrize('depth_mode,conf_mode', [('linear', ('exp', 1, float('inf'))), ('square', ('sigmoid', 0.5, 4.0)),
                                                   ('exp', None), ('linear', ('sigmoid', 0, 1))])
def test_postprocess_modes_match_oracle(cuda_device, name, depth_mode, conf_mode):
    """heads/postprocess.py:10-58: every depth mode (linear / square / exp) and confidence mode (exp / sigmoid / none) through
    both head tails (the fused DPT epilogue and the linear head's pixel-shuffle kernel)."""
    import copy
    from oracle.forward_oracle import forward_oracle
    cfg0, H, W = _small_cfgs()[name]
    cfg = copy.deepcopy(cfg0)
    cfg.depth_mode = (depth_mode, -float('inf'), float('inf'))
    cfg.conf_mode = conf_mode
    net, sd = _build(cfg, 11, cuda_device)
    imgs = synth_images(2, H, W, seed=5)
    v1 = dict(img=imgs[0]['img'].to(cuda_device), instance=['0'])
    v2 = dict(img=imgs[1]['img'].to(cuda_device), instance=['1'])
    r1, r2 = net(v1, v2)
    o1, o2 = forward_oracle(sd, cfg, imgs[0]['img'], imgs[1]['img'])
    assert ('conf' in r1) == (conf_mode is not None) == ('conf' in o1)
    assert _rel(r1['pts3d'].cpu(), o1['pts3d']) < 3e-2 and _rel(r2['pts3d_in_other_view'].cpu(), o2['pts3d_in_other_view']) < 3e-2
    if conf_mode is not None:
        assert _rel(r1['conf'].cpu(), o1['conf']) < 3e-2 and _rel(r2['conf'].cpu(), o2['conf']) < 3e-2
        lo, hi = conf_mode[1], conf_mode[2]
        assert float(r1['conf'].min()) >= lo - 1e-6 and float(r1['conf'].max()) <= hi + 1e-6
