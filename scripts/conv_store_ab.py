"""A/B of the DPT 3x3 convolutions: 128x128 tiles with register stores (d3r_set_conv_store(0)) against the staged TMA
epilogue on 128x256 / 128x128 tiles (d3r_set_conv_store(1)), at every conv shape of the forward's DPT head for 32 pairs
of 512x384 (token grid 24x32; one head, B = 32), each with the forward's flags and addends, and cuDNN conv2d (bf16,
channels_last) on the same operands.  The two store paths are timed alternately with CUDA events over `--iters` launches
after warm-up, best of `--rounds`.  Card name, power limit and SM clocks are read with nvidia-smi before and after.

    python scripts/conv_store_ab.py [--iters 20] [--rounds 3] > out.jsonl"""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from dust3r_b200 import _lib
from dust3r_b200._lib_fwd import F_BIAS, F_RELU, F_ADD0, F_ADD1, F_OUT2_RELU
from common import card, events_ms

B = 32
LEVELS = [(96, 128), (48, 64), (24, 32), (12, 16)]   # run_dpt Hs / Ws of the 24x32 grid
LD = [96, 192, 384, 768]
SHAPES = ([(f'layer_rn{k}', H, W, LD[k], 256, F_OUT2_RELU) for k, (H, W) in enumerate(LEVELS)] +
          [(f'L{k} rcu_conv1', H, W, 256, 256, F_BIAS | F_RELU) for k, (H, W) in enumerate(LEVELS)] +
          [(f'L{k} rcu1_conv2', H, W, 256, 256, F_BIAS | F_ADD0 | F_ADD1 | F_OUT2_RELU) for k, (H, W) in enumerate(LEVELS[:3])] +
          [(f'L{k} rcu2_conv2', H, W, 256, 256, F_BIAS | F_ADD0) for k, (H, W) in enumerate(LEVELS)] +
          [('head0', 192, 256, 256, 128, F_BIAS)])


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
    print(json.dumps(dict(kind='gpu', nvidia_smi=card(dev))), flush=True)
    for name, H, W, Cin, Cout, flags in SHAPES:
        x = torch.randn((B, H, W, Cin), generator=g).bfloat16().to(dev)
        w = (torch.randn((Cout, Cin, 3, 3), generator=g) * (9 * Cin) ** -0.5).bfloat16().to(dev)
        wp = w.permute(0, 2, 3, 1).contiguous()
        bias = torch.randn((Cout,), generator=g).to(dev) if flags & F_BIAS else None
        add0 = torch.randn((B, H, W, Cout), generator=g).bfloat16().to(dev) if flags & F_ADD0 else None
        add1 = torch.randn((B, H, W, Cout), generator=g).bfloat16().to(dev) if flags & F_ADD1 else None
        out = torch.empty((B, H, W, Cout), dtype=torch.bfloat16, device=dev)
        out2 = torch.empty_like(out) if flags & F_OUT2_RELU else None
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        xc = x.permute(0, 3, 1, 2)                   # NCHW view of NHWC memory = channels_last
        wc = w.contiguous(memory_format=torch.channels_last)
        res = {}

        def run():
            _lib.check(lib.d3r_conv3x3_bf16(ptr(x), ptr(wp), ptr(out), ptr(bias), ptr(add0), ptr(add1), ptr(out2), B, H, W, Cin, Cout,
                                            flags, _lib.stream_ptr()))

        def ref():
            F.conv2d(xc, wc, padding=1)

        for store in (0, 1):
            lib.d3r_set_conv_store(store)
            events_ms(run, args.warmup, 0)
            res[store] = [t.clone() for t in (out, out2) if t is not None]
        events_ms(ref, args.warmup, 0)
        same = all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(res[0], res[1]))
        times = {0: [], 1: [], 'cudnn': []}
        for _ in range(args.rounds):
            for store in (0, 1):
                lib.d3r_set_conv_store(store)
                times[store].append(events_ms(run, args.iters, 0))
            times['cudnn'].append(events_ms(ref, args.iters, 0))
        lib.d3r_set_conv_store(1)
        flop = 2.0 * B * H * W * Cout * 9 * Cin
        best = {k: min(v) for k, v in times.items()}
        print(json.dumps(dict(kind='conv_store_ab', shape=name, B=B, H=H, W=W, Cin=Cin, Cout=Cout, flags=hex(flags), bit_identical=same,
                              register_ms=round(best[0], 4), tma_ms=round(best[1], 4), cudnn_ms=round(best['cudnn'], 4),
                              register_tflops=round(flop / best[0] / 1e9, 1), tma_tflops=round(flop / best[1] / 1e9, 1),
                              cudnn_tflops=round(flop / best['cudnn'] / 1e9, 1), speedup=round(best[0] / best[1], 3),
                              rounds={str(k): [round(t, 4) for t in v] for k, v in times.items()})), flush=True)
        del x, w, wp, add0, add1, out, out2, res
    print(json.dumps(dict(kind='gpu', nvidia_smi=card(dev))), flush=True)


if __name__ == '__main__':
    main()
