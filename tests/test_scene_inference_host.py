"""Host logic of inference() over scenes (dust3r_b200/inference.py) without a GPU: the model is a RECORDING stand-in for
encode_images / decode_pairs / forward whose "features" and "pointmaps" are plain functions of each image's pixels, and the
torch.cuda stream / event entry points inference() touches are no-ops, so everything it hands to the model can be inspected:
each distinct image is encoded once, in calls within the workspace bound; each pair is decoded once, in its (size, size)
group, in batches of at most batch_size; results land in input order with the structure of the reference's loop; and the
lists that must keep today's paths never reach encode / decode.  No kernel runs; the numerics are the `-m gpu` tests' job."""
import contextlib
import types

import pytest
import torch

import dust3r_b200.inference as inf
from dust3r_b200.image_pairs import make_pairs
from dust3r_b200.utils.device import collate_with_cat, to_cpu

E = 2


def _feat(imgs):
    """The stand-in encoder: per token, the pixel at the patch's corner (channel 0) and its square."""
    f = imgs[:, 0, ::16, ::16].float()
    return torch.stack((f, f * f), dim=-1)


def _heads(f1, f2):
    up = lambda f: f[..., 0].repeat_interleave(16, 1).repeat_interleave(16, 2)
    a, b = up(f1), up(f2)
    p1 = torch.stack((a, b.mean((1, 2), keepdim=True).expand_as(a), a + 1), dim=-1)
    p2 = torch.stack((b, a.mean((1, 2), keepdim=True).expand_as(b), b - 1), dim=-1)
    return {'pts3d': p1, 'conf': a.abs() + 1}, {'conf': b.abs() + 2, 'pts3d_in_other_view': p2}


class _Model:
    """Records every call; forward() computes what decode_pairs(encode_images(.)) computes, pair by pair."""

    def __init__(self, landscape_only=False):
        self.landscape_only = landscape_only
        self.encoded, self.decoded, self.forwarded = [], [], []

    def encode_images(self, imgs):
        self.encoded.append(imgs.clone())
        return _feat(imgs)

    def decode_pairs(self, feat1, idx1, feat2, idx2):
        self.decoded.append((tuple(feat1.shape), list(idx1), tuple(feat2.shape), list(idx2)))
        return _heads(feat1[list(idx1)], feat2[list(idx2)])

    def __call__(self, view1, view2):
        self.forwarded.append(int(view1['img'].shape[0]))
        return _heads(_feat(view1['img']), _feat(view2['img']))


class _Stream:
    def __init__(self, *a, **k):
        pass

    def wait_stream(self, s):
        pass

    def wait_event(self, e):
        pass

    def synchronize(self):
        pass


@pytest.fixture()
def fake_cuda(monkeypatch):
    """'cuda' tensors are CPU tensors, pinned memory is pageable memory, streams and events do nothing."""
    real_empty = torch.empty

    def empty(*a, pin_memory=False, device=None, **k):
        return real_empty(*a, **k)

    monkeypatch.setattr(torch, 'empty', empty)
    monkeypatch.setattr(torch.cuda, 'Stream', _Stream)
    monkeypatch.setattr(torch.cuda, 'Event', lambda *a, **k: types.SimpleNamespace(record=lambda s=None: None))
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda d=None: _Stream())
    monkeypatch.setattr(torch.cuda, 'stream', lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.Tensor, 'record_stream', lambda self, s: None)
    monkeypatch.setattr(torch.Tensor, 'cuda', lambda self, *a, **k: self, raising=False)
    real_to = torch.Tensor.to

    def to(self, *a, **k):   # keep 'cuda' tensors where they are
        if a and (a[0] == 'cuda' or isinstance(a[0], torch.device) and a[0].type == 'cuda'):
            a = a[1:]
        k.pop('device', None) if str(k.get('device', '')).startswith('cuda') else None
        return real_to(self, *a, **k) if a or k else self

    monkeypatch.setattr(torch.Tensor, 'to', to)
    return torch.device('cuda')


def _views(sizes, seed=0):
    """One view dict per image, load_images' format, every pixel of image k different from those of the others."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for k, (h, w) in enumerate(sizes):
        img = torch.rand((1, 3, h, w), generator=g) + 2 * k
        out.append(dict(img=img, true_shape=torch.tensor([[h, w]], dtype=torch.int32), idx=k, instance=str(k)))
    return out


def _loop_reference(pairs, model, dev, keep_on_device=False):
    """Today's path for mixed sizes: one pair per call (dust3r/inference.py:60-72)."""
    res = [inf.loss_of_one_batch(collate_with_cat([p]), model, None, dev) for p in pairs]
    return collate_with_cat([r if keep_on_device else to_cpu(r) for r in res], lists=True)


def _assert_same(a, b, path='out'):
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
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), path
    else:
        assert a == b, (path, a, b)


def _check_encoded_once(model, distinct, chunk):
    assert all(0 < int(t.shape[0]) <= chunk for t in model.encoded), [int(t.shape[0]) for t in model.encoded]
    got = [e for t in model.encoded for e in t]
    assert len(got) == len(distinct)
    for img in distinct:    # each distinct image exactly once
        assert sum(torch.equal(e, img[0]) for e in got) == 1


MIXED = [(64, 96), (96, 64), (64, 64), (48, 96), (64, 96), (96, 64)]


@pytest.mark.parametrize('batch_size', [1, 3, 16])
@pytest.mark.parametrize('symmetrize', [True, False])
def test_mixed_sizes_group_decode_and_keep_the_loop_structure(fake_cuda, batch_size, symmetrize):
    imgs = _views(MIXED, seed=batch_size)
    pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=symmetrize)
    model = _Model()
    out = inf.inference(pairs, model, fake_cuda, batch_size=batch_size, verbose=False)
    assert not model.forwarded
    _check_encoded_once(model, [v['img'] for v in imgs], 2 * batch_size)
    # every pair decoded once, in the group of its two sizes, batches of at most batch_size, in input order within a group
    size_of = {id(v['img']): tuple(v['img'].shape[-2:]) for v in imgs}
    seen = []
    for s1, i1, s2, i2 in model.decoded:
        assert 0 < len(i1) == len(i2) <= batch_size
        seen.extend(((s1[1] * 16, s1[2] * 16), (s2[1] * 16, s2[2] * 16)) for _ in i1)
    assert len(seen) == len(pairs)
    want = [(size_of[id(a['img'])], size_of[id(b['img'])]) for a, b in pairs]
    assert sorted(seen) == sorted(want)
    # each group's batches are full except its last one
    groups = {}
    for s1, i1, s2, i2 in model.decoded:
        groups.setdefault((s1, s2), []).append(len(i1))
    for sizes in groups.values():
        assert all(s == batch_size for s in sizes[:-1])
    _assert_same(out, _loop_reference(pairs, _Model(), fake_cuda))


@pytest.mark.parametrize('keep_on_device,return_images', [(True, True), (False, False), (True, False)])
def test_mixed_sizes_options(fake_cuda, keep_on_device, return_images):
    imgs = _views(MIXED[:4], seed=3)
    pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=True)
    out = inf.inference(pairs, _Model(), fake_cuda, batch_size=4, verbose=False, keep_on_device=keep_on_device,
                        return_images=return_images)
    ref = _loop_reference(pairs, _Model(), fake_cuda, keep_on_device=keep_on_device)
    if not return_images:
        for view in ('view1', 'view2'):
            del ref[view]['img']
    _assert_same(out, ref)


@pytest.mark.parametrize('batch_size', [1, 4, 16, 18])
@pytest.mark.parametrize('graph,symmetrize', [('complete', True), ('complete', False), ('swin-2', True), ('oneref-1', True)])
def test_same_size_scene_encodes_each_image_once(fake_cuda, batch_size, graph, symmetrize):
    imgs = _views([(64, 96)] * 7, seed=batch_size)
    pairs = make_pairs(imgs, scene_graph=graph, prefilter=None, symmetrize=symmetrize)
    model = _Model()
    out = inf.inference(pairs, model, fake_cuda, batch_size=batch_size, verbose=False)
    mb = inf._micro_batch(batch_size)
    assert not model.forwarded
    _check_encoded_once(model, [v['img'] for v in imgs], 2 * mb)
    # one decode call per micro-batch, in input order: the concatenated index lists are the pairs' images
    pos = {id(v['img']): k for k, v in enumerate(imgs)}
    assert [len(i1) for _, i1, _, _ in model.decoded] == [min(mb, len(pairs) - c) for c in range(0, len(pairs), mb)]
    i1 = [i for _, ix, _, _ in model.decoded for i in ix]
    i2 = [i for _, _, _, ix in model.decoded for i in ix]
    enc_order = [next(k for k, v in enumerate(imgs) if torch.equal(v['img'], e[None])) for t in model.encoded for e in t]
    assert [enc_order[i] for i in i1] == [pos[id(a['img'])] for a, b in pairs]
    assert [enc_order[i] for i in i2] == [pos[id(b['img'])] for a, b in pairs]
    # the stacked result equals the one-batch-per-call reference, row by row
    ref = collate_with_cat([to_cpu(inf.loss_of_one_batch(collate_with_cat(pairs[c:c + 1]), _Model(), None, fake_cuda))
                            for c in range(len(pairs))])
    for which, key in (('pred1', 'pts3d'), ('pred1', 'conf'), ('pred2', 'pts3d_in_other_view'), ('pred2', 'conf')):
        assert torch.equal(out[which][key], ref[which][key]), (which, key)
    assert torch.equal(out['view1']['img'], ref['view1']['img']) and out['view2']['idx'] == ref['view2']['idx']


def test_all_distinct_and_landscape_only_lists_keep_their_paths(fake_cuda, monkeypatch):
    # private copies of every image: the pipelined fused path, no encode / decode
    imgs = _views([(64, 96)] * 4)
    pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=True)
    private = [(dict(a, img=a['img'].clone()), dict(b, img=b['img'].clone())) for a, b in pairs]
    model = _Model()
    a = inf.inference(private, model, fake_cuda, batch_size=4, verbose=False)
    assert model.forwarded and not model.encoded and not model.decoded
    b = inf.inference(pairs, _Model(), fake_cuda, batch_size=4, verbose=False)
    for which, key in (('pred1', 'pts3d'), ('pred2', 'pts3d_in_other_view'), ('pred2', 'conf')):
        assert torch.equal(a[which][key], b[which][key])
    # landscape_only=True with mixed sizes, and view dicts of two images: today's one-call-per-batch loop
    calls = []
    real = inf.loss_of_one_batch
    monkeypatch.setattr(inf, 'loss_of_one_batch', lambda batch, m, *a, **k: calls.append(1) or real(batch, m, *a, **k))
    mixed = make_pairs(_views(MIXED[:3]), scene_graph='complete', prefilter=None, symmetrize=True)
    model = _Model(landscape_only=True)
    inf.inference(mixed, model, fake_cuda, batch_size=4, verbose=False)
    assert len(calls) == len(mixed) and not model.encoded and not model.decoded
    calls.clear()
    v = _views(MIXED)
    two = [(collate_with_cat([v[0], v[4]]), collate_with_cat([v[4], v[0]])), (collate_with_cat([v[1], v[5]]), collate_with_cat([v[0], v[4]]))]
    model = _Model()
    inf.inference(two, model, fake_cuda, batch_size=4, verbose=False)
    assert len(calls) == len(two) and not model.encoded and not model.decoded
