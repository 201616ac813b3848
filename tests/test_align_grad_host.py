"""Host side of the differentiable objective without a GPU: the C library is replaced by a recording stand-in whose
d3r_align_loss_grad writes known ramps into the gradient buffers, so the flat-to-parameter mapping of both optimizer
classes (stacked depth, per-image ParameterLists, tied focal versus fx_and_fy) and the choice between the gradient launch
and the eval_only launch can be checked on CPU tensors.  The numerics are tests/test_align_grad_gpu.py's job."""
import contextlib
import ctypes as C
import types

import numpy as np
import pytest
import torch

LOSS, LOGD0, SMALL0, ENT0 = 7.0, 0.0, 1000.0, 0.5


class _RampLib:
    """Every d3r_* entry point returns 0 and records its arguments; d3r_align_loss_grad writes
    loss = LOSS, logd_grad[k] = LOGD0 + k, small_grad[k] = SMALL0 + k, entry_loss[k] = ENT0 + k."""
    CONSTS = {'d3r_align_stream_slots_per_item': 3, 'd3r_align_stream_warps_per_cta': 8, 'd3r_align_stream_max_window': 8,
              'd3r_sizeof_align_item': 64, 'd3r_align_chunk_pixels': 2048, 'd3r_sizeof_pack_entry': 32}

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            if name == 'd3r_align_workspace_floats':
                return 4096
            if name == 'd3r_align_loss_grad':
                self._ramps(*args)
            return self.CONSTS.get(name, 0)
        return fn

    @staticmethod
    def _ramps(desc_ref, logd_ptr, small_ptr, ent_ptr, stream):
        d = desc_ref._obj
        n, E = d.n_imgs, d.n_edges
        n_pix = (C.c_int64 * (n + 1)).from_address(d.img_pix_off)[n]
        (C.c_float * 1).from_address(d.loss_out)[0] = LOSS
        for ptr, count, base in ((logd_ptr, n_pix, LOGD0), (small_ptr, 11 * n + 10 * E, SMALL0), (ent_ptr, 2 * E, ENT0)):
            if ptr:
                np.frombuffer((C.c_float * count).from_address(ptr), dtype=np.float32)[:] = base + np.arange(count)


@pytest.fixture()
def ramp_lib(monkeypatch):
    from dust3r_b200 import _lib
    lib = _RampLib()
    cpu = torch.device('cpu')
    monkeypatch.setattr(_lib, 'require_cuda_device', lambda d: cpu)
    monkeypatch.setattr(_lib, 'get_lib', lambda: lib)
    monkeypatch.setattr(_lib, 'check', lambda rc: None)
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda d=None: types.SimpleNamespace(cuda_stream=0, synchronize=lambda: None))
    monkeypatch.setattr(torch.cuda, 'get_device_properties', lambda d: types.SimpleNamespace(multi_processor_count=148))
    monkeypatch.setattr(torch.Tensor, 'is_cuda', property(lambda t: True))     # the engine asserts device-resident log-depths
    return lib


SHAPES = [(8, 8), (4, 12), (8, 4)]
EDGES = [(0, 1), (1, 2), (2, 0), (0, 2)]


def _scene(cls, **kw):
    g = torch.Generator().manual_seed(0)
    p1 = [torch.randn(SHAPES[i] + (3,), generator=g) for i, j in EDGES]
    p2 = [torch.randn(SHAPES[j] + (3,), generator=g) for i, j in EDGES]
    c1 = [1 + torch.rand(SHAPES[i], generator=g) for i, j in EDGES]
    c2 = [1 + torch.rand(SHAPES[j], generator=g) for i, j in EDGES]
    view1, view2 = dict(idx=[i for i, j in EDGES]), dict(idx=[j for i, j in EDGES])
    return cls(view1, view2, dict(pts3d=p1, conf=c1), dict(pts3d_in_other_view=p2, conf=c2), verbose=False, **kw)


def _flat_small_grads(n, E):
    """The ramp split the way the C ABI lays out `small`: poses n*7 | focals n*2 | pp n*2 | pw_poses E*8 | adaptors E*2."""
    s = SMALL0 + torch.arange(11 * n + 10 * E, dtype=torch.float32)
    o = np.cumsum([0, 7 * n, 2 * n, 2 * n, 8 * E, 2 * E])
    return (s[o[0]:o[1]].view(n, 7), s[o[1]:o[2]].view(n, 2), s[o[2]:o[3]].view(n, 2), s[o[3]:o[4]].view(E, 8),
            s[o[4]:o[5]].view(E, 2))


def test_stacked_optimizer_gradient_mapping(ramp_lib):
    from dust3r_b200.cloud_opt.optimizer import PointCloudOptimizer
    net = _scene(PointCloudOptimizer, optimize_pp=True)
    n, E, A = 3, len(EDGES), 64
    net.pw_adaptors.requires_grad_(True)
    loss = net()
    assert loss.requires_grad and float(loss.detach()) == LOSS
    loss.backward()
    poses, focals, pp, pw, adapt = _flat_small_grads(n, E)
    assert torch.equal(net.im_depthmaps.grad, LOGD0 + torch.arange(n * A, dtype=torch.float32).view(n, A))   # pixel stride max_area
    assert torch.equal(net.im_poses.grad, poses)
    assert net.im_focals.grad.shape == (n, 1) and torch.equal(net.im_focals.grad, focals[:, :1])           # tied focal: slot 0
    assert torch.equal(net.im_pp.grad, pp) and torch.equal(net.pw_poses.grad, pw) and torch.equal(net.pw_adaptors.grad, adapt)
    assert [c[0] for c in ramp_lib.calls].count('d3r_align_loss_grad') == 1


@pytest.mark.parametrize('fx_and_fy', [False, True])
def test_modular_optimizer_gradient_mapping(ramp_lib, fx_and_fy):
    from dust3r_b200.cloud_opt.modular_optimizer import ModularPointCloudOptimizer
    net = _scene(ModularPointCloudOptimizer, fx_and_fy=fx_and_fy)
    n, E = 3, len(EDGES)
    net.im_poses[1].requires_grad_(False)          # a frozen camera gets no gradient
    (2 * net()).backward()
    poses, focals, pp, pw, adapt = _flat_small_grads(n, E)
    off = 0
    for i, (H, W) in enumerate(SHAPES):                # depth maps packed back to back, no padding
        assert torch.equal(net.im_depthmaps[i].grad, 2 * (LOGD0 + torch.arange(off, off + H * W, dtype=torch.float32)).view(H, W))
        off += H * W
        if i == 1:
            assert net.im_poses[i].grad is None
        else:
            assert torch.equal(net.im_poses[i].grad, 2 * poses[i])
        assert torch.equal(net.im_focals[i].grad, 2 * (focals[i] if fx_and_fy else focals[i, :1]))
        assert net.im_pp[i].grad is None               # principal points are not optimised by default
    assert torch.equal(net.pw_poses.grad, 2 * pw) and net.pw_adaptors.grad is None


def test_modular_ret_details_and_stacked_refusal(ramp_lib):
    from dust3r_b200.cloud_opt.modular_optimizer import ModularPointCloudOptimizer
    from dust3r_b200.cloud_opt.optimizer import PointCloudOptimizer
    net = _scene(ModularPointCloudOptimizer)
    with torch.no_grad():
        loss, details = net(ret_details=True)
    E = len(EDGES)
    assert not loss.requires_grad and float(loss) == LOSS and details.device.type == 'cpu' and details.shape == (3, 3)
    want = -torch.ones((3, 3))
    for e, (i, j) in enumerate(EDGES):
        want[i, j] = float((np.float32(ENT0 + 2 * e) + np.float32(ENT0 + 2 * e + 1)) * np.float32(E))
    assert torch.equal(details, want)
    with pytest.raises(NotImplementedError):
        _scene(PointCloudOptimizer)(ret_details=True)


@pytest.mark.parametrize('cls_name', ['PointCloudOptimizer', 'ModularPointCloudOptimizer'])
def test_no_grad_forward_is_an_eval_only_run(ramp_lib, cls_name):
    from dust3r_b200.cloud_opt import modular_optimizer, optimizer
    cls = getattr(optimizer if cls_name == 'PointCloudOptimizer' else modular_optimizer, cls_name)
    net = _scene(cls)
    with torch.no_grad():
        loss = net()
    assert not loss.requires_grad
    for p in net.parameters():                         # frozen parameters: no graph even in grad mode
        p.requires_grad_(False)
    net()
    names = [c[0] for c in ramp_lib.calls]
    assert 'd3r_align_loss_grad' not in names
    runs = [args for name, args in ramp_lib.calls if name == 'd3r_align_run']
    assert len(runs) == 2 and all(args[0]._obj.eval_only == 1 and args[1:3] == (0, 1) for args in runs)
