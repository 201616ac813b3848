"""Host logic of the sharded global alignment (distributed.shard_images, distributed.global_aligner_sharded and the sharded
AlignEngine) without a GPU: the C library is replaced by a recording stand-in, the torch.cuda entry points by no-ops, and the
collectives run over gloo process groups of 2 and 3 spawned ranks on CPU tensors.  What is checked is what every rank hands
to the kernels and to the collectives -- its pack table, its work items, the per-iteration order pixel pass -> all-reduce
of the accumulator block -> small step, and the broadcasts at the start and end of a run.  No kernel runs; the numerics are
tests/test_align_sharded_gpu.py's job."""
import contextlib
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

N_WS = 1 << 16          # workspace floats the stand-in reports
RB_OFF = 16             # where the stand-in puts the all-reduce block (floats)


class _RecordingLib:
    """Every d3r_* entry point returns 0 and records its name and arguments; the size queries answer like the library."""
    CONSTS = {'d3r_align_stream_slots_per_item': 3, 'd3r_align_stream_warps_per_cta': 8, 'd3r_align_stream_max_window': 8,
              'd3r_sizeof_align_item': 64, 'd3r_align_chunk_pixels': 2048, 'd3r_sizeof_pack_entry': 32}

    def __init__(self):
        self.calls = []
        self.pack_tables = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            if name == 'd3r_align_workspace_floats':
                return N_WS
            if name == 'd3r_align_reduce_block':
                n, E, off, words = args
                off._obj.value, words._obj.value = RB_OFF, 26 * E + 12 * n + 1
            if name == 'd3r_align_pack_entries':      # the table only lives as long as the call
                from dust3r_b200.cloud_opt.engine import PACK_ENTRY
                buf = (C.c_char * (args[1] * PACK_ENTRY.itemsize)).from_address(args[0])
                self.pack_tables.append(np.frombuffer(buf, dtype=PACK_ENTRY).copy())
            return self.CONSTS.get(name, 0)
        return fn


def _fake_cuda(setattr_):
    """Routes the engine's library and torch.cuda calls to the stand-in (setattr_ is monkeypatch.setattr or setattr)."""
    from dust3r_b200 import _lib
    lib = _RecordingLib()
    cpu = torch.device('cpu')
    setattr_(_lib, 'require_cuda_device', lambda d: cpu)
    setattr_(_lib, 'get_lib', lambda: lib)
    setattr_(_lib, 'check', lambda rc: None)
    setattr_(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    setattr_(torch.cuda, 'current_stream', lambda d=None: types.SimpleNamespace(cuda_stream=0, synchronize=lambda: None))
    setattr_(torch.cuda, 'get_device_properties', lambda d: types.SimpleNamespace(multi_processor_count=4))
    return lib


@pytest.fixture()
def fake_cuda(monkeypatch):
    return _fake_cuda(monkeypatch.setattr)


# scenes: (image shapes, edges).  Mixed sizes (multiples of 4 pixels, partial last slots), a complete graph, and a graph
# with fewer images than the 3-rank group has ranks.
SCENES = {
    'mixed': ([(24, 32), (32, 24), (16, 48), (24, 32), (20, 36)], [(0, 1), (1, 0), (2, 0), (3, 2), (1, 3), (4, 1), (2, 4)]),
    'n8': ([(32, 48)] * 8, [(i, j) for i in range(8) for j in range(i)]),
    'n2': ([(16, 32), (16, 16)], [(0, 1)]),
}


def _degrees(n, edges):
    deg = [0] * n
    for i, j in edges:
        deg[i] += 1
        deg[j] += 1
    return deg


def _inputs(shapes, edges):
    g = torch.Generator().manual_seed(0)
    pred_i = [torch.randn(shapes[i] + (3,), generator=g) for i, j in edges]
    pred_j = [torch.randn(shapes[j] + (3,), generator=g) for i, j in edges]
    conf_i = [1 + torch.rand(shapes[i], generator=g) for i, j in edges]
    conf_j = [1 + torch.rand(shapes[j], generator=g) for i, j in edges]
    return pred_i, pred_j, conf_i, conf_j


def _engine(shapes, edges, **kw):
    from dust3r_b200.cloud_opt.engine import AlignEngine
    pred_i, pred_j, conf_i, conf_j = _inputs(shapes, edges)
    eng = AlignEngine(edges, shapes, pred_i, pred_j, conf_i, conf_j, 'cpu', variant='per_edge', **kw)
    return eng, (pred_i, pred_j)


def _item_slots(eng):
    """(image, 64-pixel slot) of every slot of every work item of the engine."""
    from dust3r_b200.cloud_opt.engine import ITEM
    if eng.n_items == 0:
        return []
    arr = eng._items.numpy().view(ITEM)
    return [(int(r['img']), int(r['slot0']) + s) for r in arr for s in range(int(r['nslots']))]


# ---------------------------------------------------------------------------------------------- shard_images
@pytest.mark.parametrize('scene', list(SCENES))
@pytest.mark.parametrize('world', [1, 2, 3, 4, 7])
def test_shard_images_contiguous_complete_balanced(scene, world):
    from dust3r_b200.cloud_opt.engine import SLOT_PX, stream_cost
    from dust3r_b200.distributed import shard_images
    shapes, edges = SCENES[scene]
    deg = _degrees(len(shapes), edges)
    shards = shard_images(shapes, deg, world)
    assert shards == shard_images(list(shapes), list(deg), world)                 # deterministic, pure
    assert len(shards) == world and shards[0][0] == 0 and shards[-1][1] == len(shapes)
    assert all(a <= b for a, b in shards) and all(shards[r][1] == shards[r + 1][0] for r in range(world - 1))
    cost = stream_cost([(h * w + SLOT_PX - 1) // SLOT_PX for h, w in shapes], deg)
    even = cost.sum() / world
    for a, b in shards:
        assert abs(cost[a:b].sum() - even) <= cost.max() + 1e-9, (shards, cost)
    if len(shapes) < world:
        assert sum(1 for a, b in shards if a == b) >= world - len(shapes)


def test_shard_images_uses_the_streaming_cost():
    """A heavy image (many entries) gets a rank of its own; equal images split evenly."""
    from dust3r_b200.distributed import shard_images
    assert shard_images([(64, 64)] * 8, [7] * 8, 2) == [(0, 4), (4, 8)]
    assert shard_images([(64, 64)] * 4, [97, 1, 1, 1], 2) == [(0, 1), (1, 4)]
    assert sum(a == b for a, b in shard_images([(8, 8)] * 2, [1, 1], 4)) == 2      # two idle ranks


# ---------------------------------------------------------------------------------------------- sharded engine, gloo
def _worker(rank, world, port, scene, niter, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        lib = _fake_cuda(setattr)
        from dust3r_b200.distributed import shard_images
        shapes, edges = SCENES[scene]
        shards = shard_images(shapes, _degrees(len(shapes), edges), world)
        eng, (pred_i, pred_j) = _engine(shapes, edges, shards=shards)
        # which entry every packed row reads: the pointer of its pointmap
        ptr_entry = {}
        for e in range(len(edges)):
            ptr_entry[pred_i[e].data_ptr()] = int(eng._edge_ent[e, 0])
            ptr_entry[pred_j[e].data_ptr()] = int(eng._edge_ent[e, 1])
        packs = lib.pack_tables
        rows = [(ptr_entry[int(r['pts'])], int(r['obs_off']), int(r['area'])) for t in packs for r in t]

        # collectives are recorded into the same sequence as the library calls
        ws0 = eng.workspace.data_ptr()
        real_ar, real_bc = dist.all_reduce, dist.broadcast

        def all_reduce(t, op=None, group=None, **kw):
            lib.calls.append(('all_reduce', (str(t.dtype), t.numel(), (t.data_ptr() - ws0) // 4, op == dist.ReduceOp.SUM)))
            return real_ar(t, op=op, group=group, **kw)

        def broadcast(t, src, group=None, **kw):
            lib.calls.append(('broadcast', (src, t.numel())))
            return real_bc(t, src=src, group=group, **kw)
        dist.all_reduce, dist.broadcast = all_reduce, broadcast
        eng.logd = torch.full((int(eng.pix_off[-1]),), float(rank))
        eng.small.fill_(float(rank))
        del lib.calls[:]
        eng.run(niter)
        seq = [(name, args if name in ('all_reduce', 'broadcast') else args[1:-1]) for name, args in lib.calls
               if name in ('all_reduce', 'broadcast', 'd3r_align_pixel_pass', 'd3r_align_small_step', 'd3r_align_prepare')]
        q.put((rank, dict(shards=shards, owned=eng.owned, rows=rows, n_packs=len(packs), slots=_item_slots(eng),
                          n_items=eng.n_items, total_obs=eng.total_obs, seq=seq, logd=eng.logd.numpy().copy(),
                          small=eng.small.numpy().copy(), reduce_block=eng.reduce_block, window=eng.stream_window)))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _run_ranks(world, scene, niter):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 31000 + (os.getpid() % 1500) + 7 * world
    procs = [ctx.Process(target=_worker, args=(r, world, port, scene, niter, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return [got[r] for r in range(world)]


@pytest.mark.parametrize('world,scene', [(2, 'mixed'), (2, 'n8'), (3, 'mixed'), (3, 'n2')])
def test_sharded_engine_tables_and_collectives(fake_cuda, world, scene):
    shapes, edges = SCENES[scene]
    n, E = len(shapes), len(edges)
    niter = 3
    ref, _ = _engine(shapes, edges)                       # the single-rank engine of the same scene
    ent_ptr = ref._ent_ptr.numpy()
    ranks = _run_ranks(world, scene, niter)
    words = 26 * E + 12 * n + 1
    all_slots = []
    for rank, got in enumerate(ranks):
        lo, hi = got['owned']
        assert got['shards'][rank] == (lo, hi) and got['shards'] == ranks[0]['shards']
        # pack table: exactly this rank's entries in CSR order, observation offsets local to the rank
        assert [k for k, _, _ in got['rows']] == list(range(ent_ptr[lo], ent_ptr[hi]))
        assert got['n_packs'] == (1 if hi > lo else 0)
        off = 0
        for k, obs_off, area in got['rows']:
            img = int(np.searchsorted(ent_ptr, k, side='right') - 1)
            assert lo <= img < hi and area == shapes[img][0] * shapes[img][1] and obs_off == off
            off += -(-area // 64) * 64
        assert got['total_obs'] == off
        assert all(lo <= img < hi for img, _ in got['slots']) and (got['n_items'] > 0) == (hi > lo)
        assert got['window'] == ref.stream_window                   # every rank's small step picks the same version
        all_slots += got['slots']
        # the collectives and the launches, in order
        assert got['reduce_block'] == (RB_OFF, words)
        seq = got['seq']
        assert seq[0] == ('broadcast', (0, int(ref.pix_off[-1]) + ref.n_small))       # rank 0's parameters, once
        assert seq[1][0] == 'd3r_align_prepare'
        body = seq[2:2 + niter * (3 if hi > lo else 2)]
        per_it = (['d3r_align_pixel_pass'] if hi > lo else []) + ['all_reduce', 'd3r_align_small_step']
        for it in range(niter):
            chunk = body[it * len(per_it):(it + 1) * len(per_it)]
            assert [name for name, _ in chunk] == per_it
            for name, args in chunk:
                assert args == (('torch.int64', words, RB_OFF, True) if name == 'all_reduce' else (it,))
        tail = seq[2 + len(body):]
        owners = [(r, a, b) for r, (a, b) in enumerate(got['shards']) if b > a]
        assert tail == [('broadcast', (r, int(ref.pix_off[b] - ref.pix_off[a]))) for r, a, b in owners]
        # parameters after the run: rank 0's on every rank (the stand-in kernels change nothing)
        assert (got['logd'] == 0).all() and (got['small'] == 0).all()
    # across the ranks the items cover every (image, slot) -- hence every (entry, slot) -- of the single-rank table once
    assert sorted(all_slots) == sorted(_item_slots(ref)) and len(set(all_slots)) == len(all_slots)


def test_sharded_engine_refuses_the_general_kernel(fake_cuda, monkeypatch):
    monkeypatch.setattr(dist, 'get_world_size', lambda group=None: 2)
    monkeypatch.setattr(dist, 'get_rank', lambda group=None: 0)
    with pytest.raises(ValueError, match='streaming kernel'):
        _engine([(5, 7), (9, 3)], [(0, 1), (1, 0)], shards=[(0, 1), (1, 2)])
    with pytest.raises(ValueError, match='streaming kernel'):
        _engine([(8, 8), (8, 8)], [(0, 1), (1, 0)], shards=[(0, 1), (1, 2)], kernel='general')


def test_sharded_engine_has_no_differentiable_objective(fake_cuda, monkeypatch):
    monkeypatch.setattr(dist, 'get_world_size', lambda group=None: 2)
    monkeypatch.setattr(dist, 'get_rank', lambda group=None: 1)
    eng, _ = _engine([(8, 8), (8, 8)], [(0, 1), (1, 0)], shards=[(0, 1), (1, 2)])
    assert eng.owned == (1, 2)
    with pytest.raises(NotImplementedError):
        eng.loss_and_grad()


# ---------------------------------------------------------------------------------------------- public entry point
def _dust3r_output(n=3, H=8, W=16):
    from dust3r_b200.utils.synth import synth_pair_predictions
    edges = [(i, j) for i in range(n) for j in range(n) if i != j]
    return synth_pair_predictions(n, edges, H, W, seed=0)


def test_global_aligner_sharded_without_a_process_group_is_global_aligner(monkeypatch):
    import dust3r_b200.cloud_opt as cloud_opt
    from dust3r_b200.cloud_opt import GlobalAlignerMode
    from dust3r_b200.distributed import global_aligner_sharded
    assert not dist.is_initialized()
    seen = []
    sentinel = object()

    def fake(out, device, mode=None, **kw):
        seen.append((out, device, mode, kw))
        return sentinel
    monkeypatch.setattr(cloud_opt, 'global_aligner', fake)
    out = _dust3r_output()
    mode = GlobalAlignerMode.ModularPointCloudOptimizer
    assert global_aligner_sharded(out, 'cpu', mode=mode, verbose=False) is sentinel
    assert seen == [(out, 'cpu', mode, dict(verbose=False))]


def test_global_aligner_sharded_in_a_group_of_one_builds_no_shards():
    from dust3r_b200.cloud_opt import PointCloudOptimizer
    from dust3r_b200.distributed import global_aligner_sharded
    dist.init_process_group('gloo', store=dist.HashStore(), rank=0, world_size=1)
    try:
        torch.manual_seed(0)
        scene = global_aligner_sharded(_dust3r_output(), 'cpu', verbose=False)
        assert type(scene) is PointCloudOptimizer and '_align_shard' not in scene.__dict__
    finally:
        dist.destroy_process_group()


def test_global_aligner_sharded_scene_carries_this_ranks_shards(monkeypatch):
    """In a group of several ranks the scene remembers every rank's image range; a copy (mask_sky) shares it."""
    import copy
    from dust3r_b200.cloud_opt import GlobalAlignerMode, ModularPointCloudOptimizer
    from dust3r_b200.distributed import global_aligner_sharded, shard_images
    monkeypatch.setattr(dist, 'is_initialized', lambda: True)
    monkeypatch.setattr(dist, 'get_world_size', lambda group=None: 2)
    out = _dust3r_output(n=4)
    scene = global_aligner_sharded(out, 'cpu', mode=GlobalAlignerMode.ModularPointCloudOptimizer, verbose=False)
    assert type(scene) is ModularPointCloudOptimizer
    shard = scene._align_shard
    assert shard.shards == shard_images(scene.imshapes, [6] * 4, 2) and shard.group is None
    assert copy.deepcopy(scene)._align_shard is shard
    viewer = global_aligner_sharded(_dust3r_output(n=2), 'cpu', mode=GlobalAlignerMode.PairViewer, verbose=False)
    assert '_align_shard' not in viewer.__dict__
