"""Host logic of inference() over scenes (dust3r_b200/inference.py) without a GPU: the model is a RECORDING stand-in for
encode_images / decode_pairs / forward whose "features" and "pointmaps" are plain functions of each image's pixels, and the
torch.cuda stream / event entry points inference() touches are no-ops, so everything it hands to the model can be inspected:
each distinct image is encoded once, in calls within the workspace bound; each pair is decoded once, in its (size, size)
group, in batches of at most one micro-batch; results land in input order with the structure of the reference's loop; and
the lists forward() has to check or handle never reach encode / decode.  No kernel runs; the numerics are the `-m gpu`
tests' job."""
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
        self.decoded.append((feat1, list(idx1), feat2, list(idx2)))
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


PINNED = []   # shapes of the pinned buffers allocated under fake_cuda


@pytest.fixture()
def fake_cuda(monkeypatch):
    """'cuda' tensors are CPU tensors, pinned memory is pageable memory (its allocations recorded in PINNED), streams and
    events do nothing."""
    real_empty = torch.empty
    PINNED.clear()

    def empty(*a, pin_memory=False, device=None, **k):
        t = real_empty(*a, **k)
        if pin_memory:
            PINNED.append(tuple(t.shape))
        return t

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


def _staged_images(chunk):
    """Pinned image buffers (n,3,H,W) allocated so far hold at most one encode call's images."""
    assert all(s[0] <= chunk for s in PINNED if len(s) == 4 and s[1] == 3), PINNED


def _positions(feat, imgs):
    """Position in `imgs` of the image behind each row of the stand-in features `feat`."""
    return [next(k for k, v in enumerate(imgs) if torch.equal(_feat(v['img'])[0], f)) for f in feat]


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
    mb = inf._micro_batch(batch_size)
    assert not model.forwarded
    _check_encoded_once(model, [v['img'] for v in imgs], 2 * mb)
    # every pair decoded once, in the group of its two sizes, batches of at most mb, in input order within a group
    size_of = {id(v['img']): tuple(v['img'].shape[-2:]) for v in imgs}
    seen = []
    for f1, i1, f2, i2 in model.decoded:
        assert 0 < len(i1) == len(i2) <= mb
        seen.extend(((f1.shape[1] * 16, f1.shape[2] * 16), (f2.shape[1] * 16, f2.shape[2] * 16)) for _ in i1)
    assert len(seen) == len(pairs)
    want = [(size_of[id(a['img'])], size_of[id(b['img'])]) for a, b in pairs]
    assert sorted(seen) == sorted(want)
    # each group's batches are full except its last one
    groups = {}
    for f1, i1, f2, i2 in model.decoded:
        groups.setdefault((f1.shape, f2.shape), []).append(len(i1))
    for sizes in groups.values():
        assert all(s == mb for s in sizes[:-1])
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
        _staged_images(2 * inf._micro_batch(4))
    _assert_same(out, ref)


KEYS = (('pred1', 'pts3d'), ('pred1', 'conf'), ('pred2', 'pts3d_in_other_view'), ('pred2', 'conf'))


@pytest.mark.parametrize('batch_size', [1, 4, 16, 18])
@pytest.mark.parametrize('graph,symmetrize', [('complete', True), ('complete', False), ('swin-2', True), ('oneref-1', True)])
@pytest.mark.parametrize('scenes', [1, 2])
def test_same_size_scene_encodes_each_image_once(fake_cuda, batch_size, graph, symmetrize, scenes):
    # with two scenes the list is the pairs of one followed by those of the other, which shares no image with it
    imgs = [_views([(64, 96)] * 7, seed=batch_size + 100 * s) for s in range(scenes)]
    per_scene = [make_pairs(v, scene_graph=graph, prefilter=None, symmetrize=symmetrize) for v in imgs]
    imgs, pairs = sum(imgs, []), sum(per_scene, [])
    model = _Model()
    out = inf.inference(pairs, model, fake_cuda, batch_size=batch_size, verbose=False)
    mb = inf._micro_batch(batch_size)
    assert not model.forwarded
    _check_encoded_once(model, [v['img'] for v in imgs], 2 * mb)
    # each scene is decoded in calls of one micro-batch, in input order: the concatenated index lists are the pairs' images
    pos = {id(v['img']): k for k, v in enumerate(imgs)}
    assert [len(i1) for _, i1, _, _ in model.decoded] == [min(mb, len(p) - c) for p in per_scene for c in range(0, len(p), mb)]
    assert [k for f, ix, _, _ in model.decoded for k in _positions(f[ix], imgs)] == [pos[id(a['img'])] for a, b in pairs]
    assert [k for _, _, f, ix in model.decoded for k in _positions(f[ix], imgs)] == [pos[id(b['img'])] for a, b in pairs]
    # no encode call, and no feature tensor handed to a decode call, holds images of both scenes
    for t in model.encoded:
        assert len({k // 7 for k in _positions(_feat(t), imgs)}) == 1
    for f1, _, f2, _ in model.decoded:
        assert len({k // 7 for k in _positions(torch.cat((f1, f2)), imgs)}) == 1
    # the stacked result equals the one-batch-per-call reference, row by row
    ref = collate_with_cat([to_cpu(inf.loss_of_one_batch(collate_with_cat(pairs[c:c + 1]), _Model(), None, fake_cuda))
                            for c in range(len(pairs))])
    for which, key in KEYS:
        assert torch.equal(out[which][key], ref[which][key]), (which, key)
    assert torch.equal(out['view1']['img'], ref['view1']['img']) and out['view2']['idx'] == ref['view2']['idx']
    # without the images in the result, pageable images are staged one encode call at a time
    PINNED.clear()
    bare = inf.inference(pairs, _Model(), fake_cuda, batch_size=batch_size, verbose=False, return_images=False)
    _staged_images(2 * mb)
    assert 'img' not in bare['view1'] and all(torch.equal(bare[which][key], out[which][key]) for which, key in KEYS)


@pytest.mark.parametrize('batch_size', [4, 18])
def test_private_copies_are_encoded_a_micro_batch_at_a_time(fake_cuda, batch_size):
    """Private copies of every image share nothing, so every group is mb pairs: one encode call of its view-1 then view-2
    images and one decode call -- the calls forward() makes on a micro-batch -- with the result of the shared list."""
    imgs = _views([(64, 96)] * 4)
    pairs = make_pairs(imgs, scene_graph='complete', prefilter=None, symmetrize=True)
    private = [(dict(a, img=a['img'].clone()), dict(b, img=b['img'].clone())) for a, b in pairs]
    model = _Model()
    a = inf.inference(private, model, fake_cuda, batch_size=batch_size, verbose=False)
    mb, n = inf._micro_batch(batch_size), len(private)
    assert not model.forwarded
    assert [len(i1) for _, i1, _, _ in model.decoded] == [min(mb, n - c) for c in range(0, n, mb)]
    assert len(model.encoded) == len(model.decoded)
    for t, c in zip(model.encoded, range(0, n, mb)):
        assert torch.equal(t, torch.cat([p[0]['img'] for p in private[c:c + mb]] + [p[1]['img'] for p in private[c:c + mb]]))
    _assert_same(a, inf.inference(pairs, _Model(), fake_cuda, batch_size=batch_size, verbose=False))


def test_view_dicts_of_several_images_are_taken_row_by_row(fake_cuda):
    v = _views([(64, 96)] * 6, seed=5)
    d = [collate_with_cat(v[c:c + 2]) for c in range(0, 6, 2)]
    pairs = [(d[a], d[b]) for a in range(3) for b in range(3) if a != b]
    model = _Model()
    out = inf.inference(pairs, model, fake_cuda, batch_size=4, verbose=False)
    assert not model.forwarded
    _check_encoded_once(model, [x['img'] for x in v], 2 * inf._micro_batch(4))
    ref = collate_with_cat([to_cpu(inf.loss_of_one_batch(collate_with_cat([p]), _Model(), None, fake_cuda)) for p in pairs])
    for which, key in KEYS:
        assert torch.equal(out[which][key], ref[which][key]), (which, key)
    for view in ('view1', 'view2'):
        assert torch.equal(out[view]['img'], ref[view]['img']) and out[view]['idx'] == ref[view]['idx']


@pytest.mark.parametrize('case', ['landscape_only_mixed', 'two_image_mixed', 'landscape_only_portrait_true_shape'])
def test_lists_forward_has_to_handle_take_the_loop(fake_cuda, monkeypatch, case):
    """landscape_only=True with a portrait tensor, view dicts of two images in a list of several sizes, and a shared-image
    list whose true_shape says portrait on a landscape_only=True model (a ManyAR batch): the reference's loop of forward()
    calls, one pair per call when sizes are mixed."""
    calls = []
    real = inf.loss_of_one_batch
    monkeypatch.setattr(inf, 'loss_of_one_batch', lambda batch, m, *a, **k: calls.append(1) or real(batch, m, *a, **k))
    model = _Model(landscape_only=case.startswith('landscape_only'))
    if case == 'landscape_only_mixed':
        pairs = make_pairs(_views(MIXED[:3]), scene_graph='complete', prefilter=None, symmetrize=True)
    elif case == 'two_image_mixed':
        v = _views(MIXED)
        pairs = [(collate_with_cat([v[0], v[4]]), collate_with_cat([v[4], v[0]])),
                 (collate_with_cat([v[1], v[5]]), collate_with_cat([v[0], v[4]]))]
    else:
        portrait = [dict(v, true_shape=torch.tensor([[96, 64]], dtype=torch.int32)) for v in _views([(64, 96)] * 4)]
        pairs = make_pairs(portrait, scene_graph='complete', prefilter=None, symmetrize=True)
    inf.inference(pairs, model, fake_cuda, batch_size=4, verbose=False)
    assert len(calls) == (len(pairs) if case.endswith('mixed') else -(-len(pairs) // 4))
    assert model.forwarded and not model.encoded and not model.decoded
