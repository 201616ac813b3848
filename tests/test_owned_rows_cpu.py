"""inference_sharded(keep='owned') and the scene built from its rows, on CPU: gloo groups of 2 and 3 spawned ranks, the
deterministic stand-in model of tests/test_distributed_cpu.py for the forward, and the recording stand-in for the C library
of tests/test_align_sharded_host.py for the alignment engine.  Checked: the image ranges, exactly which rows every rank
keeps and that they are bit-identical to keep='all', the one all_to_all_single and the sizes of the buffers it allocates,
im_conf, the pack table every rank hands to the kernels, and init='mst' / 'known_poses' against the all-gathered scene."""
import os
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_distributed_cpu import _FakeModel, _pairs


def _owner(shards, img):
    return next(r for r, (a, b) in enumerate(shards) if a <= img < b)


def _np(x):
    return None if x is None else x.numpy().copy()


def _pack_rows(lib, scene):
    """(dictionary, key, obs_off, area, coef) of every row of the engine's pack tables, pointers resolved to entries."""
    where = {}
    for name in ('pred_i', 'pred_j', 'conf_i', 'conf_j'):
        for key, t in getattr(scene, name).items():
            where[t.data_ptr()] = (name, key)
    return [(where[int(r['pts'])], where[int(r['conf'])], int(r['obs_off']), int(r['area']), float(r['coef']))
            for t in lib.pack_tables for r in t]


def _worker(rank, world, port, n_imgs, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from test_align_sharded_host import _fake_cuda
        from dust3r_b200.cloud_opt import GlobalAlignerMode
        from dust3r_b200.distributed import global_aligner_sharded, inference_sharded
        pairs = _pairs(n_imgs)
        full = inference_sharded(pairs, _FakeModel(), 'cpu', batch_size=2, verbose=False)
        calls = []
        real = {name: getattr(dist, name) for name in ('all_to_all_single', 'all_gather_into_tensor', 'all_gather', 'broadcast', 'all_reduce')}

        def recorder(name):
            def fn(*a, **kw):
                calls.append(name)
                return real[name](*a, **kw)
            return fn
        for name in real:
            setattr(dist, name, recorder(name))
        out = inference_sharded(pairs, _FakeModel(), 'cpu', batch_size=2, verbose=False, keep='owned')
        route_calls = list(calls)
        for name in real:
            setattr(dist, name, real[name])
        owned = out['owned']
        res = dict(shards=owned.shards, world=owned.world, imshapes=owned.imshapes, allocated=owned.allocated,
                   calls=route_calls, idx=(out['view1']['idx'], out['view2']['idx']),
                   full={(w, k): v.numpy().copy() for w in ('pred1', 'pred2') for k, v in full[w].items()},
                   kept={(w, k): [_np(x) for x in v] for w in ('pred1', 'pred2') for k, v in out[w].items()})
        # the scene of the kept rows against the scene of the all-gathered output, engines on the recording stand-in
        lib = _fake_cuda(setattr)
        mode = GlobalAlignerMode.ModularPointCloudOptimizer
        scenes = {}
        for name, o in (('all', full), ('owned', out)):
            torch.manual_seed(3)
            scenes[name] = global_aligner_sharded(o, 'cpu', mode=mode, verbose=False)
            del lib.pack_tables[:]
            scenes[name]._get_engine()
            res[f'pack_{name}'] = _pack_rows(lib, scenes[name])
            res[f'im_conf_{name}'] = [c.detach().numpy().copy() for c in scenes[name].im_conf]
        res['dict_keys'] = {name: sorted(getattr(scenes['owned'], name).keys()) for name in ('pred_i', 'pred_j', 'conf_i', 'conf_j')}
        q.put((rank, res))
        dist.barrier()
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def _run(world, n_imgs, worker=_worker):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 35000 + (os.getpid() % 1500) + 11 * world + (n_imgs % 7)
    procs = [ctx.Process(target=worker, args=(r, world, port, n_imgs, q)) for r in range(world)]
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


# (world, images): complete symmetrised graphs; 2 images over 3 ranks (a rank without images and one without pairs); one
# pair over 2 ranks (rank 1 computes no pair)
@pytest.mark.parametrize('world,n_imgs', [(2, 5), (3, 5), (3, 4), (3, 2), (2, -2)])
def test_owned_rows(world, n_imgs):
    from dust3r_b200.distributed import shard_bounds, shard_images
    pairs = _pairs(n_imgs)
    edges = [(int(a['idx']), int(b['idx'])) for a, b in pairs]
    n = 1 + max(max(e) for e in edges)
    deg = np.bincount(np.asarray(edges).reshape(-1), minlength=n)
    shards = shard_images([(16, 32)] * n, deg.tolist(), world)
    ranks = _run(world, n_imgs)
    E = len(edges)
    row_floats = 2 * 4 * 16 * 32          # [pts3d | conf | pts3d_in_other_view | conf]
    for rank, got in enumerate(ranks):
        assert got['shards'] == shards and got['world'] == world and got['imshapes'] == [(16, 32)] * n
        assert got['idx'] == ([i for i, j in edges], [j for i, j in edges])
        # one collective, and no buffer of the full list's size
        assert got['calls'] == ['all_to_all_single'], got['calls']
        assert [a[0] for a in got['allocated']] == ['send', 'recv']
        plo, phi = shard_bounds(E, world, rank)
        assert got['allocated'][0][2] <= 4 * (phi - plo) * row_floats * 3 // 2       # each row once, a view-2 half twice
        if E > 1:
            assert all(b < 4 * E * row_floats for _, _, b in got['allocated'])
        lo, hi = shards[rank]
        kept_floats = 0
        for e, (i, j) in enumerate(edges):
            whole, half = lo <= i < hi, lo <= j < hi
            for (w, k), rows in got['kept'].items():
                v = rows[e]
                if whole or (half and w == 'pred2'):
                    assert v is not None and np.array_equal(v, got['full'][(w, k)][e]), (rank, e, w, k)
                    kept_floats += v.size
                else:
                    assert v is None, (rank, e, w, k)
        assert got['allocated'][1][2] == 4 * kept_floats        # the receive buffer holds the kept rows and nothing else
        # the scene holds exactly the kept entries; im_conf and the engine's pack table are those of the all-gathered scene
        keys_i = sorted('%d_%d' % (i, j) for i, j in edges if lo <= i < hi)
        keys_j = sorted('%d_%d' % (i, j) for i, j in edges if lo <= i < hi or lo <= j < hi)
        assert got['dict_keys'] == dict(pred_i=keys_i, conf_i=keys_i, pred_j=keys_j, conf_j=keys_j)
        assert all(np.array_equal(a, b) for a, b in zip(got['im_conf_owned'], got['im_conf_all']))
        assert got['pack_owned'] == got['pack_all'] and len(got['pack_owned']) == int(deg[lo:hi].sum())
    # every row is kept by the owner of its first image, every view-2 half also by the owner of its second image
    for e, (i, j) in enumerate(edges):
        keepers = [r for r in range(world) if ranks[r]['kept'][('pred1', 'pts3d')][e] is not None]
        assert keepers == [_owner(shards, i)]
        halves = {r for r in range(world) if ranks[r]['kept'][('pred2', 'pts3d_in_other_view')][e] is not None}
        assert halves == {_owner(shards, i), _owner(shards, j)}


def owned_output(out, device='cpu'):
    """What inference_sharded(keep='owned') returns on this rank, for a full inference() result `out` (any mix of image
    sizes): this rank's slice of the pairs routed by PairOutputRoute, as inference_sharded routes its forward's output."""
    from dust3r_b200.cloud_opt.commons import get_imshapes
    from dust3r_b200.distributed import OwnedRows, PairOutputRoute, shard_bounds, shard_images
    edges = list(zip(out['view1']['idx'], out['view2']['idx']))
    p1, p2 = out['pred1'], out['pred2']
    imshapes = get_imshapes(edges, p1['pts3d'], p2['pts3d_in_other_view'])
    degrees = np.bincount(np.asarray(edges).reshape(-1), minlength=len(imshapes)).tolist()
    world, rank = dist.get_world_size(), dist.get_rank()
    shards = shard_images(imshapes, degrees, world)
    lo, hi = shard_bounds(len(edges), world, rank)
    comm = torch.device(device) if dist.get_backend() == 'nccl' else torch.device('cpu')
    route = PairOutputRoute(edges, imshapes, shards, True, comm)
    route.pack(*({k: [t.to(device) for t in v[lo:hi]] for k, v in p.items()} for p in (p1, p2)))
    k1, k2 = route.exchange(device)
    return dict(view1=out['view1'], view2=out['view2'], pred1=k1, pred2=k2, loss=None,
                owned=OwnedRows(shards, world, imshapes, route.allocated))


def _init_worker(rank, world, port, n_imgs, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from test_align_sharded_host import _fake_cuda
        from dust3r_b200.cloud_opt import GlobalAlignerMode, init_im_poses
        from dust3r_b200.distributed import global_aligner_sharded
        from dust3r_b200.utils.synth import synth_consistent_scene
        _fake_cuda(setattr)
        edges = [(i, j) for i in range(n_imgs) for j in range(n_imgs) if i != j]
        full, cams, f = synth_consistent_scene(n_imgs, edges, 16, 24, seed=5)
        trees = []
        real_mst = init_im_poses.minimum_spanning_tree

        def mst(*a, **kw):
            res = real_mst(*a, **kw)
            trees.append(res[1])
            return res
        init_im_poses.minimum_spanning_tree = mst
        res = {}
        for init in ('mst', 'known_poses'):
            for name, o in (('all', full), ('owned', owned_output(full))):
                torch.manual_seed(11 + rank)
                scene = global_aligner_sharded(o, 'cpu', mode=GlobalAlignerMode.ModularPointCloudOptimizer, verbose=False)
                if init == 'mst':
                    init_im_poses.init_minimum_spanning_tree(scene)
                else:
                    scene.preset_pose(cams)
                    scene.preset_focal([f] * n_imgs)
                    init_im_poses.init_from_known_poses(scene, min_conf_thr=scene.min_conf_thr)
                res[(init, name)] = dict(pw=scene.pw_poses.detach().numpy().copy(),
                                         depth=[d.detach().numpy().copy() for d in scene.im_depthmaps],
                                         poses=scene.get_im_poses().detach().numpy(), focals=scene.get_focals().detach().numpy())
        res['trees'] = trees
        q.put((rank, res))
        dist.barrier()
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 3])
def test_owned_scene_initialisation_equals_all_gathered(world):
    """init='mst' and 'known_poses' on kept rows: the same spanning tree and, on the CPU, the same initial pairwise poses,
    depth maps, poses and focals bit for bit on the rank that keeps each edge / owns each image."""
    ranks = _run(world, 5, worker=_init_worker)
    for got in ranks:
        assert got['trees'][0] == got['trees'][1] == ranks[0]['trees'][0]
        for init in ('mst', 'known_poses'):
            a, b = got[(init, 'all')], got[(init, 'owned')]
            if init == 'mst':       # every rank holds the walk's result
                for k in ('poses', 'focals'):
                    assert np.array_equal(a[k], b[k]), (init, k)
            assert all(np.array_equal(x, y) for x, y in zip(a['depth'], b['depth'])), init
            assert np.array_equal(a['pw'], b['pw']), init


def test_owned_output_refused_by_other_entry_points(monkeypatch):
    """global_aligner and a group of another size refuse the kept rows; PairViewer needs every pair."""
    from dust3r_b200.cloud_opt import GlobalAlignerMode, global_aligner
    from dust3r_b200.distributed import OwnedRows, global_aligner_sharded
    from dust3r_b200.utils.synth import synth_pair_predictions
    out = synth_pair_predictions(2, [(0, 1), (1, 0)], 8, 16, seed=0)
    out['owned'] = OwnedRows([(0, 1), (1, 2)], 2, [(8, 16)] * 2)
    with pytest.raises(ValueError, match='global_aligner_sharded'):
        global_aligner(out, 'cpu', verbose=False)
    with pytest.raises(ValueError, match='group of 2 ranks'):
        global_aligner_sharded(out, 'cpu', verbose=False)        # no process group: a group of one
    monkeypatch.setattr(dist, 'is_initialized', lambda: True)
    monkeypatch.setattr(dist, 'get_world_size', lambda group=None: 2)
    with pytest.raises(ValueError, match='PairViewer'):
        global_aligner_sharded(out, 'cpu', mode=GlobalAlignerMode.PairViewer, verbose=False)
    with pytest.raises(ValueError, match="'all' or 'owned'"):
        from dust3r_b200.distributed import inference_sharded
        inference_sharded([], None, 'cpu', keep='some')
