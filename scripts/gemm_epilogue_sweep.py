"""Epilogue-cost sweep of the wgmma GEMM: same shape, different fused epilogues (iteration aid)."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dust3r_b200 import _lib
from scripts.forward_quick_bench import timeit

lib = _lib.get_lib()
CASES = [(49152, 4096, 1024, (1, 3, 5)), (49152, 3072, 1024, (1, 3)), (49152, 1024, 1024, (1, 9, 0x11)),
         (24576, 768, 768, (1, 9, 0x11)), (49152, 1024, 4096, (1, 0x11)), (24576, 3072, 768, (1, 3)),
         (24576, 768, 3072, (0x11,)), (24576, 2304, 768, (1,))]
import ctypes
MINKB = int(sys.argv[1]) if len(sys.argv) > 1 else 16
lib.d3r_set_gemm_pair_min_kblocks.argtypes = [ctypes.c_int32]
lib.d3r_set_gemm_pair_min_kblocks(MINKB)
for (M, N, K, flagset) in CASES:
    A = torch.randn((M, K), device='cuda').bfloat16(); B = torch.randn((N, K), device='cuda').bfloat16()
    bias = torch.randn((N,), device='cuda')
    for fl in flagset:
        out = torch.zeros((M, N), device='cuda', dtype=torch.float32 if fl & 0x18 else torch.bfloat16)
        def f():
            _lib.check(lib.d3r_gemm_bf16(A.data_ptr(), B.data_ptr(), out.data_ptr(), bias.data_ptr(), None, None, M, N, K, N, fl, None, None, 0, 0, 0, _lib.stream_ptr()))
        ms = timeit(f, warm=3, rep=10)
        print(json.dumps(dict(kind='gemm_epilogue', pair_min_kb=MINKB, M=M, N=N, K=K, flags=hex(fl), ms=round(ms, 5), tflops=round(2 * M * N * K / ms / 1e9, 1))), flush=True)
