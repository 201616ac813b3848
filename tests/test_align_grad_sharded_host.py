"""Host logic of the sharded differentiable objective (AlignEngine.sharded_loss_and_grad, behind scene() + loss.backward() on
a scene of distributed.global_aligner_sharded) without a GPU.  The C library is the recording stand-in of
tests/test_align_sharded_host.py, whose gradient entry points here write the known ramps of tests/test_align_grad_host.py:
d3r_align_grad_pixel_pass over the pixels of the images of the descriptor's work items only, d3r_align_grad_small_step (and
d3r_align_loss_grad) the loss, small-parameter and entry-loss ramps.  The collectives run over gloo groups of 1, 2 and 3 ranks
on CPU tensors.  Checked: every rank's launches and collectives in order, that the owners' broadcasts assemble the whole
log-depth gradient on every rank, that no parameter or Adam moment changes, which launch forward() picks, and the .grad and
per-edge details every rank's scene ends with.  The numerics are tests/test_align_grad_sharded_gpu.py's job."""
import ctypes as C
import os
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_align_grad_host import ENT0, LOGD0, LOSS, SMALL0, _flat_small_grads
from test_align_sharded_host import RB_OFF, SCENES, _RecordingLib, _degrees, _engine, _fake_cuda

GRAD_CALLS = ('d3r_align_prepare', 'd3r_align_grad_pixel_pass', 'd3r_align_grad_small_step', 'd3r_align_loss_grad',
              'd3r_align_pixel_pass', 'd3r_align_small_step', 'd3r_align_run')


def _floats(ptr, count):
    return np.frombuffer((C.c_float * count).from_address(ptr), dtype=np.float32)


class _GradLib(_RecordingLib):
    """The recording stand-in with ramps written by the gradient entry points (see the module docstring)."""

    def __getattr__(self, name):
        record = super().__getattr__(name)

        def fn(*args):
            rc = record(*args)
            if name == 'd3r_align_grad_pixel_pass':
                self._logd_ramp(args[0]._obj, args[1], own_items=True)
            elif name == 'd3r_align_grad_small_step':
                self._small_ramps(args[0]._obj, args[1], args[2])
            elif name == 'd3r_align_loss_grad':
                self._logd_ramp(args[0]._obj, args[1], own_items=False)
                self._small_ramps(args[0]._obj, args[2], args[3])
            return rc
        return fn

    @staticmethod
    def _logd_ramp(d, ptr, own_items):
        from dust3r_b200.cloud_opt.engine import ITEM
        n = d.n_imgs
        pix_off = np.frombuffer((C.c_int64 * (n + 1)).from_address(d.img_pix_off), dtype=np.int64)
        imgs = range(n)
        if own_items:
            items = np.frombuffer((C.c_char * (d.n_items * ITEM.itemsize)).from_address(d.items), dtype=ITEM)
            imgs = sorted({int(i) for i in items['img']})
        out = _floats(ptr, int(pix_off[n]))
        for i in imgs:
            out[pix_off[i]:pix_off[i + 1]] = LOGD0 + np.arange(pix_off[i], pix_off[i + 1])

    @staticmethod
    def _small_ramps(d, small_ptr, ent_ptr):
        n, E = d.n_imgs, d.n_edges
        _floats(d.loss_out, 1)[0] = LOSS
        _floats(small_ptr, 11 * n + 10 * E)[:] = SMALL0 + np.arange(11 * n + 10 * E)
        if ent_ptr:
            _floats(ent_ptr, 2 * E)[:] = ENT0 + np.arange(2 * E)


def _fake_grad_cuda(setattr_):
    from dust3r_b200 import _lib
    _fake_cuda(setattr_)
    lib = _GradLib()
    setattr_(_lib, 'get_lib', lambda: lib)
    setattr_(torch.Tensor, 'is_cuda', property(lambda t: True))     # the engine asserts device-resident log-depths
    return lib


def _record_collectives(lib):
    """Routes dist.all_reduce / dist.broadcast through recorders that append to lib.calls (name, (.., data pointer))."""
    real_ar, real_bc = dist.all_reduce, dist.broadcast

    def all_reduce(t, op=None, group=None, **kw):
        lib.calls.append(('all_reduce', (str(t.dtype), t.numel(), t.data_ptr(), op == dist.ReduceOp.SUM)))
        return real_ar(t, op=op, group=group, **kw)

    def broadcast(t, src, group=None, **kw):
        lib.calls.append(('broadcast', (src, t.numel(), t.data_ptr())))
        return real_bc(t, src=src, group=group, **kw)
    dist.all_reduce, dist.broadcast = all_reduce, broadcast


def _sequence(lib, eng, res):
    """The launches and collectives of lib.calls, pointers resolved to the engine's buffers and the call's results."""
    loss, logd_grad, small_grad, ent = res
    ws0, lg0 = eng.workspace.data_ptr(), logd_grad.data_ptr()
    seq = []
    for name, args in lib.calls:
        if name == 'all_reduce':
            seq.append((name, args[:2] + ((args[2] - ws0) // 4, args[3])))
        elif name == 'broadcast':
            src, numel, ptr = args
            where = (ptr - lg0) // 4 if lg0 <= ptr < lg0 + 4 * logd_grad.numel() else ('params' if numel == eng.logd.numel() + eng.n_small else ptr)
            seq.append((name, (src, numel, where)))
        elif name == 'd3r_align_grad_pixel_pass':
            seq.append((name, (args[1] == lg0,)))
        elif name == 'd3r_align_grad_small_step':
            seq.append((name, (args[0]._obj.loss_out == loss.data_ptr(), args[1] == small_grad.data_ptr(),
                               None if args[2] is None else args[2] == ent.data_ptr())))
        elif name in GRAD_CALLS:
            seq.append((name, ()))
    return seq


# ---------------------------------------------------------------------------------------------- engine, 2 and 3 ranks
def _engine_worker(rank, world, port, scene, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        lib = _fake_grad_cuda(setattr)
        from dust3r_b200.distributed import shard_images
        shapes, edges = SCENES[scene]
        shards = shard_images(shapes, _degrees(len(shapes), edges), world)
        eng, _ = _engine(shapes, edges, shards=shards)
        _record_collectives(lib)
        eng.logd = torch.full((int(eng.pix_off[-1]),), float(rank))
        eng.small.fill_(float(rank))
        eng.reset_adam()
        for k, t in enumerate((eng.logd_m, eng.logd_v, eng.small_m, eng.small_v)):
            t.fill_(10.0 * (k + 1) + rank)
        runs = {}
        for entry_loss in (False, True):
            del lib.calls[:]
            res = eng.sharded_loss_and_grad(entry_loss=entry_loss)
            runs[entry_loss] = dict(seq=_sequence(lib, eng, res), loss=float(res[0]), logd_grad=res[1].numpy().copy(),
                                    small_grad=res[2].numpy().copy(), ent=None if res[3] is None else res[3].numpy().copy())
        state = {k: getattr(eng, k).numpy().copy() for k in ('logd', 'small', 'logd_m', 'logd_v', 'small_m', 'small_v')}
        q.put((rank, dict(runs=runs, state=state, owned=eng.owned, shards=shards, words=eng.reduce_block[1],
                          n_params=int(eng.pix_off[-1]) + eng.n_small)))
        dist.barrier()
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def _run_ranks(worker, world, *args, base=38000):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = base + (os.getpid() % 1500) + 7 * world
    procs = [ctx.Process(target=worker, args=(r, world, port) + args + (q,)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        rank, res = q.get(timeout=180)
        assert not isinstance(res, str), f'rank {rank} failed:\n{res}'
        got[rank] = res
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return [got[r] for r in range(world)]


@pytest.mark.parametrize('world,scene', [(2, 'mixed'), (2, 'n8'), (3, 'mixed'), (3, 'n2')])
def test_sharded_loss_and_grad_launches_and_collectives(world, scene):
    """Per rank: rank 0's parameters broadcast, prepare, the gradient pixel pass (absent on a rank without images), the
    all-reduce of the accumulator block, the gradient small step (entry_loss only when asked for), then one broadcast of
    logd_grad per non-empty owner range.  Every rank ends with the whole log-depth gradient and untouched optimiser state."""
    shapes, edges = SCENES[scene]
    n, E = len(shapes), len(edges)
    ranks = _run_ranks(_engine_worker, world, scene)
    pix_off = np.concatenate([[0], np.cumsum([h * w for h, w in shapes])])
    assert any(a == b for a, b in ranks[0]['shards']) == (scene == 'n2')
    for rank, got in enumerate(ranks):
        lo, hi = got['owned']
        assert got['words'] == 26 * E + 12 * n + 1
        owners = [(r, a, b) for r, (a, b) in enumerate(got['shards']) if b > a]
        for entry_loss, run in got['runs'].items():
            want = [('broadcast', (0, got['n_params'], 'params')), ('d3r_align_prepare', ())]
            want += [('d3r_align_grad_pixel_pass', (True,))] if hi > lo else []
            want += [('all_reduce', ('torch.int64', got['words'], RB_OFF, True)),
                     ('d3r_align_grad_small_step', (True, True, True if entry_loss else None))]
            want += [('broadcast', (r, int(pix_off[b] - pix_off[a]), int(pix_off[a]))) for r, a, b in owners]
            assert run['seq'] == want, (rank, entry_loss)
            # the owners' slices assemble the whole gradient; the small step's outputs are the same on every rank
            assert np.array_equal(run['logd_grad'], LOGD0 + np.arange(pix_off[-1], dtype=np.float32))
            assert run['loss'] == LOSS and np.array_equal(run['small_grad'], SMALL0 + np.arange(11 * n + 10 * E, dtype=np.float32))
            assert (run['ent'] is not None) == entry_loss
            if entry_loss:
                assert np.array_equal(run['ent'], (ENT0 + np.arange(2 * E, dtype=np.float32)).reshape(E, 2))
        # the objective is rank 0's; the Adam moments are this rank's own, untouched
        st = got['state']
        assert (st['logd'] == 0).all() and (st['small'] == 0).all()
        for k, name in enumerate(('logd_m', 'logd_v', 'small_m', 'small_v')):
            assert (st[name] == 10.0 * (k + 1) + rank).all(), name


# ---------------------------------------------------------------------------------------------- scenes, 2 ranks
def _scene_output(n=5):
    from dust3r_b200.utils.synth import synth_pair_predictions
    return synth_pair_predictions(n, [(i, j) for i in range(n) for j in range(n) if i != j], 8, 16, seed=0)


def _grads(scene):
    """.grad of every optimised parameter (the observations are parameters too, and differ between kept-row scenes)."""
    kinds = ('im_depthmaps', 'im_poses', 'im_focals', 'im_pp', 'pw_poses', 'pw_adaptors')
    return {name: (None if p.grad is None else p.grad.numpy().copy()) for name, p in scene.named_parameters()
            if name.split('.')[0] in kinds}


def _scene_worker(rank, world, port, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        lib = _fake_grad_cuda(setattr)
        from test_owned_rows_cpu import owned_output
        from dust3r_b200.cloud_opt import GlobalAlignerMode
        from dust3r_b200.distributed import global_aligner_sharded
        res = {}
        for mode, kw in (('PointCloudOptimizer', dict(optimize_pp=True)), ('ModularPointCloudOptimizer', dict(fx_and_fy=True))):
            for kind in ('all', 'owned'):
                out = _scene_output() if kind == 'all' else owned_output(_scene_output())
                torch.manual_seed(7 + rank)
                scene = global_aligner_sharded(out, 'cpu', mode=GlobalAlignerMode[mode], verbose=False, **kw)
                if mode == 'ModularPointCloudOptimizer':
                    scene.im_poses[1].requires_grad_(False)
                r = dict(owned=scene._get_engine().owned)
                del lib.calls[:]
                loss = scene()
                loss.backward()
                r.update(loss=float(loss.detach()), grads=_grads(scene), calls=[c for c, _ in lib.calls if c in GRAD_CALLS])
                small = [args[2] for c, args in lib.calls if c == 'd3r_align_grad_small_step']
                r['entry_loss_passed'] = [p is not None for p in small]
                if mode == 'ModularPointCloudOptimizer':
                    del lib.calls[:]
                    with torch.no_grad():
                        _, details = scene(ret_details=True)
                    r['details'] = details.numpy().copy()
                    r['details_entry_loss'] = [args[2] is not None for c, args in lib.calls if c == 'd3r_align_grad_small_step']
                del lib.calls[:]
                with torch.no_grad():
                    scene()
                r['no_grad_calls'] = [c for c, _ in lib.calls if c in GRAD_CALLS]
                res[(mode, kind)] = r
        q.put((rank, res))
        dist.barrier()
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def test_sharded_scene_backward_and_details_on_every_rank():
    """Both optimizer classes, keep='all' and keep='owned' scenes, a frozen camera: scene() with grad on runs the sharded
    gradient (never d3r_align_loss_grad), backward() gives every rank the same .grad -- the ramps through the parameter
    mapping of the single-GPU path -- and ret_details passes an entry-loss buffer; under no_grad scene() stays the split
    eval_only iteration."""
    world = 2
    ranks = _run_ranks(_scene_worker, world, base=39600)
    n = 5
    E = n * (n - 1)
    A = 8 * 16
    poses, focals, pp, pw, adapt = (t.numpy() for t in _flat_small_grads(n, E))
    ramp = LOGD0 + np.arange(n * A, dtype=np.float32)
    for (mode, kind), r0 in ranks[0].items():
        assert ranks[1][(mode, kind)]['owned'] != r0['owned']
        for got in ranks:
            r = got[(mode, kind)]
            assert r['calls'] == ['d3r_align_prepare', 'd3r_align_grad_pixel_pass', 'd3r_align_grad_small_step'], (mode, kind)
            assert r['entry_loss_passed'] == [False] and r['loss'] == LOSS
            assert r['no_grad_calls'] == ['d3r_align_prepare', 'd3r_align_pixel_pass', 'd3r_align_small_step']
            g = r['grads']
            for name in g:
                assert (g[name] is None) == (r0['grads'][name] is None) and (g[name] is None or np.array_equal(g[name], r0['grads'][name])), name
            if mode == 'PointCloudOptimizer':
                assert np.array_equal(g['im_depthmaps'], ramp.reshape(n, A))
                assert np.array_equal(g['im_poses'], poses) and np.array_equal(g['im_focals'], focals[:, :1])
                assert np.array_equal(g['im_pp'], pp)
            else:
                for i in range(n):
                    assert np.array_equal(g[f'im_depthmaps.{i}'], ramp[i * A:(i + 1) * A].reshape(8, 16))
                    assert (g[f'im_poses.{i}'] is None) == (i == 1)
                    assert i == 1 or np.array_equal(g[f'im_poses.{i}'], poses[i])
                    assert np.array_equal(g[f'im_focals.{i}'], focals[i])
                want = -np.ones((n, n), dtype=np.float32)
                for e, (i, j) in enumerate((i, j) for i in range(n) for j in range(n) if i != j):
                    want[i, j] = (np.float32(ENT0 + 2 * e) + np.float32(ENT0 + 2 * e + 1)) * np.float32(E)
                assert r['details_entry_loss'] == [True] and np.array_equal(r['details'], want)
            assert np.array_equal(g['pw_poses'], pw) and g['pw_adaptors'] is None


# ---------------------------------------------------------------------------------------------- dispatch, one rank
@pytest.fixture()
def one_rank_group():
    dist.init_process_group('gloo', store=dist.HashStore(), rank=0, world_size=1)
    yield
    dist.destroy_process_group()


def test_forward_dispatches_on_the_scene_being_sharded(monkeypatch, one_rank_group):
    """A scene without image ranges takes the single-launch gradient, one with ranges (here over a one-rank group) the
    sharded one; both hand the same gradients to the same parameters.  loss_and_grad keeps refusing a sharded engine and
    sharded_loss_and_grad refuses an engine without ranges."""
    from dust3r_b200.cloud_opt import GlobalAlignerMode, global_aligner
    from dust3r_b200.distributed import _AlignShard
    lib = _fake_grad_cuda(monkeypatch.setattr)
    grads, calls = [], []
    for sharded in (False, True):
        torch.manual_seed(0)
        scene = global_aligner(_scene_output(), 'cpu', mode=GlobalAlignerMode.ModularPointCloudOptimizer, verbose=False)
        if sharded:
            scene._align_shard = _AlignShard([(0, scene.n_imgs)], None)
        del lib.calls[:]
        scene().backward()
        calls.append([c for c, _ in lib.calls if c in GRAD_CALLS])
        grads.append(_grads(scene))
        eng = scene._get_engine()
        with pytest.raises(NotImplementedError if sharded else ValueError):
            (eng.loss_and_grad if sharded else eng.sharded_loss_and_grad)()
    assert calls == [['d3r_align_prepare', 'd3r_align_loss_grad'],
                     ['d3r_align_prepare', 'd3r_align_grad_pixel_pass', 'd3r_align_grad_small_step']]
    assert grads[0].keys() == grads[1].keys()
    for name, g in grads[0].items():
        assert (g is None and grads[1][name] is None) or np.array_equal(g, grads[1][name]), name
