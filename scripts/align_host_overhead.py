"""Host-side overhead of the alignment e2e call (global_aligner + compute_global_alignment, BASELINE configs[2]) measured
WITHOUT a GPU: the C library and the torch.cuda entry points the engine uses are replaced by no-ops and everything runs on CPU
tensors, so what is timed is exactly the Python / numpy / torch-CPU work that surrounds the kernel launches on an H100.

    python -O scripts/align_host_overhead.py        # -O: the engine asserts that its buffers are CUDA tensors

Recorded in this container (DESIGN.md section 3): constructor 14-15 ms (7 ms = the reference's seeded torch.randn depth draws,
4 ms per-image confidence maxima, 3-4 ms parameter registration), engine build + tables + launch loop 5 ms."""
import sys, time, types, contextlib, cProfile, pstats
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from dust3r_b200 import _lib
import ctypes as C

class FakeFn:
    def __init__(self, name, ret=0): self.name, self.ret = name, ret
    def __call__(self, *a): return self.ret
class FakeLib:
    def __getattr__(self, name):
        ret = {'d3r_align_stream_slots_per_item': 3, 'd3r_align_stream_warps_per_cta': 8, 'd3r_align_stream_max_window': 8,
               'd3r_sizeof_align_item': 64, 'd3r_align_chunk_pixels': 2048, 'd3r_align_workspace_floats': 100000,
               'd3r_sizeof_align_desc': C.sizeof(_lib.AlignDesc), 'd3r_sizeof_pack_entry': 32}.get(name, 0)
        return FakeFn(name, ret)
class FakeStream:
    cuda_stream = 0
    def synchronize(self): pass


def main():
    cpu = torch.device('cpu')
    _lib.require_cuda_device = lambda d: cpu
    fake = FakeLib()
    _lib.get_lib = lambda: fake
    _lib.check = lambda rc: None
    torch.cuda.device = lambda d: contextlib.nullcontext()
    torch.cuda.current_stream = lambda d=None: FakeStream()
    torch.cuda.get_device_properties = lambda d: types.SimpleNamespace(multi_processor_count=132)
    torch.cuda.synchronize = lambda *a: None

    from dust3r_b200.utils.synth import synth_pair_predictions
    from dust3r_b200.cloud_opt import global_aligner
    n, H, W = 8, 384, 512
    edges = [(i, j) for i in range(n) for j in range(i)]
    out = synth_pair_predictions(n, edges, H, W, seed=0)

    def once():
        torch.manual_seed(0)
        net = global_aligner(out, 'cpu', verbose=False)
        t1 = time.perf_counter()
        loss = net.compute_global_alignment(init=None, niter=300, schedule='cosine', lr=0.01)
        return net, t1
    for k in range(3):
        t0 = time.perf_counter(); net, t1 = once(); t2 = time.perf_counter()
        print('ctor %.1f ms   compute %.1f ms' % ((t1 - t0) * 1e3, (t2 - t1) * 1e3))
    pr = cProfile.Profile(); pr.enable(); once(); pr.disable()
    pstats.Stats(pr).sort_stats('cumulative').print_stats(35)


if __name__ == '__main__':
    main()
