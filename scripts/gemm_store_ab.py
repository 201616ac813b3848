"""A/B of the projection GEMMs' epilogue store path: register stores (d3r_set_gemm_store(0)) against the staged TMA
store / TMA reduce-add (d3r_set_gemm_store(1)), on the eight projection shapes of the forward (32 pairs of 512x384:
64 encoder images and 32 decoder passes per side of 768 tokens), each with the epilogue the forward uses there, and
torch.matmul (cuBLAS, bf16 output) on the same operands.  The two store paths are timed alternately, with CUDA events
over `--iters` launches after warm-up.  Card name, power limit and SM clocks are read with nvidia-smi queries.

    python scripts/gemm_store_ab.py [--iters 20] [--rounds 3] > out.jsonl"""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from dust3r_b200 import _lib
from dust3r_b200._lib_fwd import F_BIAS, F_GELU, F_RESID_INPLACE, F_ROPE
from oracle.forward_oracle import rope_tables
from common import card, events_ms

ENC, DEC = 64 * 768, 32 * 768
SHAPES = [('enc qkv', ENC, 3072, 1024, 'rope'), ('enc proj', ENC, 1024, 1024, 'resid'), ('enc fc1', ENC, 4096, 1024, 'gelu'),
          ('enc fc2', ENC, 1024, 4096, 'resid'), ('dec qkv', DEC, 2304, 768, 'rope'), ('dec proj', DEC, 768, 768, 'resid'),
          ('dec fc1', DEC, 3072, 768, 'gelu'), ('dec fc2', DEC, 768, 3072, 'resid')]
GH, GW = 24, 32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    _lib.require_cuda_device(dev)
    lib = _lib.get_lib()
    g = torch.Generator(device='cpu').manual_seed(0)
    cos, sin = (t.to(dev).contiguous() for t in rope_tables(64, max(GH, GW), 100.0))
    print(json.dumps(dict(kind='gpu', nvidia_smi=card(dev))), flush=True)
    for name, M, N, K, epi in SHAPES:
        A = torch.randn((M, K), generator=g).bfloat16().to(dev)
        B = (torch.randn((N, K), generator=g) * K ** -0.5).bfloat16().to(dev)
        bias = torch.randn((N,), generator=g).to(dev)
        if epi == 'resid':
            out = torch.randn((M, N), generator=g).to(dev)
            flags = F_BIAS | F_RESID_INPLACE
        else:
            out = torch.empty((M, N), dtype=torch.bfloat16, device=dev)
            flags = F_BIAS | (F_GELU if epi == 'gelu' else F_ROPE)
        rope = (C.c_void_p(cos.data_ptr()), C.c_void_p(sin.data_ptr()), 2 * N // 3, GH * GW, GW) if epi == 'rope' else (None, None, 0, 0, 0)

        def run():
            _lib.check(lib.d3r_gemm_bf16(A.data_ptr(), B.data_ptr(), out.data_ptr(), bias.data_ptr(), None, None, M, N, K, N, flags,
                                         *rope, _lib.stream_ptr()))

        def ref():
            torch.matmul(A, B.T)

        times = {0: [], 1: [], 'torch': []}
        for store in (0, 1):
            lib.d3r_set_gemm_store(store)
            events_ms(run, args.warmup, 0)
        events_ms(ref, args.warmup, 0)
        for _ in range(args.rounds):
            for store in (0, 1):
                lib.d3r_set_gemm_store(store)
                times[store].append(events_ms(run, args.iters, 0))
            times['torch'].append(events_ms(ref, args.iters, 0))
        lib.d3r_set_gemm_store(1)
        flop = 2.0 * M * N * K
        best = {k: min(v) for k, v in times.items()}
        print(json.dumps(dict(kind='gemm_store_ab', shape=name, M=M, N=N, K=K, epilogue=epi,
                              register_ms=round(best[0], 4), tma_ms=round(best[1], 4), torch_ms=round(best['torch'], 4),
                              register_tflops=round(flop / best[0] / 1e9, 1), tma_tflops=round(flop / best[1] / 1e9, 1),
                              torch_tflops=round(flop / best['torch'] / 1e9, 1), speedup=round(best[0] / best[1], 3),
                              rounds={str(k): [round(t, 4) for t in v] for k, v in times.items()})), flush=True)
        del A, B, out
    print(json.dumps(dict(kind='gpu', nvidia_smi=card(dev))), flush=True)


if __name__ == '__main__':
    main()
