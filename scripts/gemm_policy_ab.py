"""A/B of the GEMM kernel-family policy on the whole forward step (B = 32 pairs, 512x384, ViT-L / DPT), interleaved."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from dust3r_b200 import _lib
from scripts.forward_quick_bench import timeit
from bench import build_model, H, W
lib = _lib.get_lib()
net, cfg = build_model(torch.device('cuda:0'))
packed = net.repack()
B = 32
imgs = torch.rand((2 * B, 3, H, W), device='cuda') * 2 - 1
idx1, idx2 = np.arange(B, dtype=np.int32), B + np.arange(B, dtype=np.int32)
f = lambda: packed.forward(imgs, idx1, idx2, B, H, W)
timeit(f, warm=3, rep=5)
for rnd in range(2):
    for name, impl, kb in (('pair>=16kb', 2, 16), ('pair>=12kb', 2, 12), ('pair>=4kb', 2, 4), ('pair always', 1, 16)):
        lib.d3r_set_gemm_impl(impl); lib.d3r_set_gemm_pair_min_kblocks(kb)
        ms = timeit(f, warm=2, rep=6)
        print(json.dumps(dict(policy=name, ms=round(ms, 3), pairs_per_s=round(B / ms * 1e3, 1))), flush=True)
