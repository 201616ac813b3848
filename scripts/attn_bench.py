"""Attention kernel A/B timing (iteration aid): impl 2 (P through shared memory) vs impl 3 (P in registers) on the model's shapes."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dust3r_b200 import _lib
from scripts.forward_quick_bench import timeit
lib = _lib.get_lib()
for (B, Hh, N) in [(64, 16, 768), (32, 12, 768)]:
    ld = 3 * Hh * 64
    qkv = torch.randn((B, N, ld), device='cuda').bfloat16()
    out = torch.empty((B, N, Hh * 64), device='cuda', dtype=torch.bfloat16)
    res = {}
    for impl in (2, 3):   # impl 2 (P through smem), impl 3 (P in registers)
        lib.d3r_set_attention_impl(impl)
        def f():
            _lib.check(lib.d3r_attention_hd64(qkv.data_ptr(), ld, qkv.data_ptr() + Hh * 128, ld, qkv.data_ptr() + Hh * 256, ld,
                                              out.data_ptr(), Hh * 64, B, Hh, N, N, 0.125, _lib.stream_ptr()))
        ms = timeit(f, warm=3, rep=20)
        res[impl] = out.float().clone()
        print(json.dumps(dict(kind='attention', impl=impl, B=B, heads=Hh, N=N, ms=round(ms, 4), tflops=round(4 * B * Hh * N * N * 64 / ms / 1e9, 1))), flush=True)
    print(json.dumps(dict(kind='attention_diff', max_abs_2_vs_3=float((res[2] - res[3]).abs().max()))), flush=True)
lib.d3r_set_attention_impl(3)
