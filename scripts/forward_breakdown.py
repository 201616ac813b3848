"""Per-launch breakdown of one forward step (32 pairs, ViT-L/DPT 512x384): aggregates the library's per-launch
CUDA-event records by (kernel, shape/flags).  Usage: python scripts/forward_breakdown.py [B] > out.jsonl"""
import sys, os, json, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from bench import build_model, H, W
from common import card
from dust3r_b200 import _lib


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    dev = torch.device('cuda:0')
    net, cfg = build_model(dev)
    packed = net.repack()
    imgs = torch.rand((2 * B, 3, H, W), device='cuda') * 2 - 1
    idx1, idx2 = np.arange(B, dtype=np.int32), B + np.arange(B, dtype=np.int32)
    for _ in range(3):
        packed.forward(imgs, idx1, idx2, B, H, W)
    torch.cuda.synchronize()
    _lib.prof_enable(True)
    packed.forward(imgs, idx1, idx2, B, H, W)
    torch.cuda.synchronize()
    recs = _lib.prof_dump()
    _lib.prof_enable(False)
    agg = collections.OrderedDict()
    for r in recs:
        k = (r['tag'], r['detail'])
        a = agg.setdefault(k, dict(n=0, ms=0.0, flops=0.0, bytes=0.0))
        a['n'] += 1; a['ms'] += r['ms']; a['flops'] += r['flops']; a['bytes'] += r['bytes']
    tot = sum(a['ms'] for a in agg.values())
    print(json.dumps(dict(kind='forward_breakdown', B=B, total_ms=tot, card=card(dev))))
    for (tag, det), a in sorted(agg.items(), key=lambda kv: -kv[1]['ms']):
        print(json.dumps(dict(tag=tag, detail=det, n=a['n'], ms=round(a['ms'], 4), share=round(a['ms'] / tot, 4),
                              tflops=round(a['flops'] / a['ms'] / 1e9, 1) if a['flops'] else None,
                              gbs=round(a['bytes'] / a['ms'] / 1e6, 1) if a['bytes'] else None)))


if __name__ == '__main__':
    main()
