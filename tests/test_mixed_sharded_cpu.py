"""inference_sharded on pair lists of several image sizes, on CPU: gloo groups of 2 and 3 spawned ranks and a stand-in model
that returns a geometrically consistent pointmap pair of each pair's own sizes.  Checked on every rank: keep='all' is
single-process inference() entry for entry and bit for bit, with the entries of the gather sharing one storage; keep='owned'
keeps exactly the rows PairOutputRoute assigns, equal to routing inference()'s result; init='mst' on the kept rows matches
it on the all-gathered output (alignment engines on the recording stand-in of tests/test_align_sharded_host.py); and a
list of one size still goes through PairOutputGather."""
import math
import os
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _pose(k):
    """Rotation rows and translation of camera k (camera to world): cameras on a small arc."""
    a = 0.2 * (k - 2)
    c, s = math.cos(a), math.sin(a)
    return ((c, 0.0, s), (0.0, 1.0, 0.0), (-s, 0.0, c)), (1.5 * s, 0.05 * k, 0.3 * (1 - c))


def _affine(R, t, p):
    x, y, z = p.unbind(-1)
    return torch.stack([R[r][0] * x + R[r][1] * y + R[r][2] * z + t[r] for r in range(3)], dim=-1)


def _cloud(img):
    """Points of one image (3, H, W) in its own camera's frame: depth from the first channel, focal 1.2 max(H, W)."""
    H, W = img.shape[-2:]
    f = 1.2 * max(H, W)
    v, u = torch.meshgrid(*(torch.arange(n, dtype=torch.float32, device=img.device) for n in (H, W)), indexing='ij')
    depth = 2.5 + 0.4 * img[0]
    return torch.stack(((u - W / 2) * depth / f, (v - H / 2) * depth / f, depth), dim=-1)


class _SceneModel:
    """Pair (i, j) -> image i's points in camera i's frame and image j's points moved into camera i's frame (plus 1 % of
    noise), each at its own image's size, on the images' device.  Every item of a batch is computed alone with elementwise
    operations, so its bits do not depend on the batch it is computed in."""
    conf_mode = ('exp', 1, float('inf'))

    def __call__(self, view1, view2):
        out = dict(pts3d=[], conf=[]), dict(pts3d_in_other_view=[], conf=[])
        for b in range(view1['img'].shape[0]):
            i, j = int(view1['idx'][b]), int(view2['idx'][b])
            a, c = view1['img'][b], view2['img'][b]
            (Ri, ti), (Rj, tj) = _pose(i), _pose(j)
            world = _affine(Rj, tj, _cloud(c))
            in_i = _affine(tuple(zip(*Ri)), (0.0, 0.0, 0.0), world - torch.tensor(ti, device=c.device))
            # a little pair-dependent noise, so that the scene's alignment loss has a floor above zero
            out[0]['pts3d'].append(_cloud(a) + 0.01 * torch.sin(5 * a + j).permute(1, 2, 0))
            in_i = in_i + 0.01 * torch.sin(3 * c + i).permute(1, 2, 0)
            out[0]['conf'].append(1.5 + 2 * (a[1] + 1))
            out[1]['pts3d_in_other_view'].append(in_i)
            out[1]['conf'].append(1.5 + 2 * (c[2] + 1))
        if self.conf_mode is None:
            for o in out:
                del o['conf']
        return tuple({k: torch.stack(v) for k, v in o.items()} for o in out)


class _SceneModelNoConf(_SceneModel):
    conf_mode = None


SIZES3 = [(16, 24), (24, 16), (16, 32), (16, 24), (24, 16)]


def _views(sizes):
    from dust3r_b200.utils.synth import synth_images
    return [dict(synth_images(1, h, w, seed=30 + k)[0], idx=k, instance=str(k)) for k, (h, w) in enumerate(sizes)]


def _graph(name):
    """The pair lists: 'complete5' = complete symmetrised on 5 images of 3 sizes; 'uniform_first' = the 6 pairs of three
    images of one size first (rank 0's slice is of one size at world 2 and 3), then pairs with two images of other sizes;
    'two_images' = 2 images of two sizes, 2 pairs (a rank without pairs at world 3); 'same' = 4 images of one size."""
    from dust3r_b200.image_pairs import make_pairs
    if name == 'complete5':
        return make_pairs(_views(SIZES3), scene_graph='complete', prefilter=None, symmetrize=True)
    if name == 'uniform_first':
        v = _views([(16, 24)] * 3 + [(24, 16), (16, 32)])
        ij = [(0, 1), (1, 0), (0, 2), (2, 0), (1, 2), (2, 1), (0, 3), (3, 0), (1, 4), (4, 1), (3, 4), (4, 3)]
        return [(v[i], v[j]) for i, j in ij]
    if name == 'two_images':
        return make_pairs(_views([(16, 24), (24, 16)]), scene_graph='complete', prefilter=None, symmetrize=True)
    return make_pairs(_views([(16, 24)] * 4), scene_graph='complete', prefilter=None, symmetrize=True)


def _assert_same(a, b, path='out'):
    """Same structure (types, keys, list lengths), same values bit for bit, same dtypes and devices.  Keys are compared as
    dict equality compares them, in any order: the forward names a pointmap last when it renames it."""
    assert type(a) is type(b), (path, type(a), type(b))
    if isinstance(a, dict):
        assert sorted(a) == sorted(b), (path, list(a), list(b))
        for k in a:
            _assert_same(a[k], b[k], f'{path}.{k}')
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), (path, len(a), len(b))
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, f'{path}[{i}]')
    elif torch.is_tensor(a):
        assert a.dtype == b.dtype and a.shape == b.shape and a.device == b.device, (path, a.dtype, b.dtype, a.shape, b.shape)
        assert torch.equal(a, b), path
    else:
        assert a == b, (path, a, b)


def _no_img(out):
    return dict(out, **{v: {k: x for k, x in out[v].items() if k != 'img'} for v in ('view1', 'view2')})


def _check_all(pairs, model, ref, calls):
    """keep='all' against inference(), for return_images True and False; one all-gather; one storage for the entries."""
    from dust3r_b200.distributed import inference_sharded
    for return_images in (True, False):
        del calls[:]
        out = inference_sharded(pairs, model, 'cpu', batch_size=2, verbose=False, return_images=return_images)
        assert calls == ['all_gather_into_tensor'], calls
        _assert_same(out, ref if return_images else _no_img(ref))
        entries = [t for p in ('pred1', 'pred2') for v in out[p].values() for t in v]
        assert len({t.untyped_storage().data_ptr() for t in entries}) == 1
    return out


def _check_owned(pairs, model, full, ref, calls):
    """keep='owned': the rows of PairOutputRoute's rule, equal to the all-gathered entries and to routing inference()."""
    from test_owned_rows_cpu import owned_output
    from dust3r_b200.distributed import inference_sharded, pair_graph, shard_images
    del calls[:]
    out = inference_sharded(pairs, model, 'cpu', batch_size=2, verbose=False, keep='owned')
    assert calls == ['all_to_all_single'], calls
    edges, imshapes = pair_graph(pairs)
    degrees = np.bincount(np.asarray(edges).reshape(-1), minlength=len(imshapes)).tolist()
    world, rank = dist.get_world_size(), dist.get_rank()
    shards = shard_images(imshapes, degrees, world)
    owned = out['owned']
    assert owned.shards == shards and owned.world == world and owned.imshapes == imshapes
    lo, hi = shards[rank]
    for which in ('pred1', 'pred2'):
        assert sorted(out[which]) == sorted(full[which])
        for key, rows in out[which].items():
            assert len(rows) == len(edges)
            for e, (i, j) in enumerate(edges):
                if lo <= i < hi or (which == 'pred2' and lo <= j < hi):
                    _assert_same(rows[e], full[which][key][e], f'{which}.{key}[{e}]')
                else:
                    assert rows[e] is None, (which, key, e)
    _assert_same(out['view1'], ref['view1'])
    _assert_same(out['view2'], ref['view2'])
    if 'conf' in ref['pred1']:      # routing inference()'s result (the stand-in route of test_owned_rows_cpu has confidences)
        routed = owned_output(ref)
        assert routed['owned'].shards == shards and routed['owned'].imshapes == imshapes
        for which in ('pred1', 'pred2'):
            for key, rows in routed[which].items():
                for e, t in enumerate(rows):
                    assert (t is None) == (out[which][key][e] is None), (which, key, e)
                    if t is not None:
                        assert torch.equal(t, out[which][key][e]), (which, key, e)
    return out


def _mst(full, owned):
    """init='mst' on the all-gathered output and on the kept rows: spanning trees, pairwise poses, depth maps, poses, focals."""
    from test_align_sharded_host import _fake_cuda
    from dust3r_b200.cloud_opt import GlobalAlignerMode, init_im_poses
    from dust3r_b200.distributed import global_aligner_sharded
    _fake_cuda(setattr)
    trees = []
    real_mst = init_im_poses.minimum_spanning_tree

    def mst(*a, **kw):
        res = real_mst(*a, **kw)
        trees.append(res[1])
        return res
    init_im_poses.minimum_spanning_tree = mst
    res = {}
    for name, o in (('all', full), ('owned', owned)):
        torch.manual_seed(11 + dist.get_rank())
        scene = global_aligner_sharded(o, 'cpu', mode=GlobalAlignerMode.ModularPointCloudOptimizer, verbose=False)
        init_im_poses.init_minimum_spanning_tree(scene)
        res[name] = dict(pw=scene.pw_poses.detach().numpy().copy(), depth=[d.detach().numpy().copy() for d in scene.im_depthmaps],
                         poses=scene.get_im_poses().detach().numpy(), focals=scene.get_focals().detach().numpy())
    init_im_poses.minimum_spanning_tree = real_mst
    assert len(trees) == 2 and trees[0] == trees[1]
    a, b = res['all'], res['owned']
    assert np.isfinite(a['poses']).all() and np.isfinite(a['focals']).all()
    for k in ('poses', 'focals', 'pw'):
        assert np.array_equal(a[k], b[k]), k
    assert all(np.array_equal(x, y) for x, y in zip(a['depth'], b['depth']))
    return trees[0], a['pw']


def _worker(rank, world, port, graph, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from dust3r_b200 import distributed
        from dust3r_b200.inference import inference
        calls = []
        real = {name: getattr(dist, name) for name in ('all_to_all_single', 'all_gather_into_tensor', 'all_gather', 'broadcast', 'all_reduce')}

        def recorder(name):
            def fn(*a, **kw):
                calls.append(name)
                return real[name](*a, **kw)
            return fn
        for name in real:
            setattr(dist, name, recorder(name))
        pairs = _graph(graph)
        res = {}
        if graph == 'same':     # one size: the stacked layout of PairOutputGather, as before
            used = []

            class Spy(distributed.PairOutputGather):
                def __init__(self, *a, **kw):
                    used.append(a)
                    super().__init__(*a, **kw)
            distributed.PairOutputGather = Spy
            out = distributed.inference_sharded(pairs, _SceneModel(), 'cpu', batch_size=2, verbose=False)
            assert len(used) == 1 and calls == ['all_gather_into_tensor'], (used, calls)
            _assert_same(out, inference(pairs, _SceneModel(), 'cpu', batch_size=2, verbose=False))
            assert all(torch.is_tensor(v) and v.shape[0] == len(pairs) for p in ('pred1', 'pred2') for v in out[p].values())
        else:
            for model in (_SceneModelNoConf(), _SceneModel()):
                ref = inference(pairs, model, 'cpu', batch_size=2, verbose=False)
                assert isinstance(ref['pred1']['pts3d'], list)
                full = _check_all(pairs, model, ref, calls)
                owned = _check_owned(pairs, model, full, ref, calls)
            for name in real:
                setattr(dist, name, real[name])
            res['tree'], res['pw'] = _mst(full, owned)     # the outputs of the model with confidences
        q.put((rank, res))
        dist.barrier()
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def _run(world, graph):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 37000 + (os.getpid() % 1500) + 13 * world + ('complete5', 'uniform_first', 'two_images', 'same').index(graph)
    procs = [ctx.Process(target=_worker, args=(r, world, port, graph, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        rank, res = q.get(timeout=300)
        assert not isinstance(res, str), f'rank {rank} failed:\n{res}'
        got[rank] = res
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return [got[r] for r in range(world)]


@pytest.mark.parametrize('graph', ['complete5', 'uniform_first', 'two_images'])
@pytest.mark.parametrize('world', [2, 3])
def test_mixed_sizes_sharded(world, graph):
    ranks = _run(world, graph)
    for got in ranks:       # every rank builds the same spanning tree and ends with the same pairwise poses
        assert got['tree'] == ranks[0]['tree'] and np.array_equal(got['pw'], ranks[0]['pw'])


def test_one_size_keeps_the_stacked_gather():
    _run(2, 'same')


def test_row_layout(monkeypatch):
    """The row layout every rank computes from the pair list alone: per-rank float counts, padding to the largest, and a
    view dict of several images counting as that many rows."""
    from dust3r_b200.distributed import MixedPairOutputGather, row_shapes
    pairs = _graph('uniform_first')
    shapes, pair_rows = row_shapes(pairs)
    assert pair_rows == [1] * 12 and shapes[6] == ((16, 24), (24, 16))
    two = dict(img=torch.zeros((2, 3, 8, 8)))
    assert row_shapes([(two, two)]) == ([((8, 8), (8, 8))] * 2, [2])
    floats = [4 * (a[0] * a[1] + b[0] * b[1]) for a, b in shapes]

    monkeypatch.setattr(dist, 'get_world_size', lambda group=None: 3)
    monkeypatch.setattr(dist, 'get_rank', lambda group=None: 0)
    g = MixedPairOutputGather(shapes, pair_rows, True, 'cpu')
    assert g.rows == [(0, 4), (4, 8), (8, 12)]
    assert g.counts == [sum(floats[0:4]), sum(floats[4:8]), sum(floats[8:12])] and g.width == max(g.counts)
    assert g.start[4:8] == [0] + np.cumsum(floats[4:7]).tolist()
    assert MixedPairOutputGather(shapes, pair_rows, False, 'cpu').counts == [c * 3 // 4 for c in g.counts]
