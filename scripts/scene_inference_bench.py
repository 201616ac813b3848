"""Multi-view inference() through the public API on the published ViT-L / DPT architecture (synthetic weights): pairs/s,
encoder passes and algorithmic work of whole scenes.

Cases (synthetic views, make_pairs complete graph, symmetrised):
  sym50_bs1    50 views at 512x384, 2450 pairs, batch_size 1 (the demo's value)
  sym50_bs32   the same list, batch_size 32
  mixed12_bs16 12 views, 6 at 512x384 and 6 at 384x512, 132 pairs, batch_size 16

Encoder passes are counted at the library calls (images handed to an encoder pass); algorithmic work is
passes x 523.05 GFLOP + pairs x 810.7 GFLOP (DESIGN.md §4: 1046.1 GFLOP of encoder per pair of 512x384 images, 437.3 of
decoders and 373.4 of heads; a 384x512 image has as many tokens).  Each case warms up on its first 64 pairs (on all of
them with two sizes), then runs `--repeat` timed times, each ending in a device synchronise; one JSON line per case.
`--dump-outputs DIR` stores a fixed sample of every case's last result, for output-for-output comparison of two builds.

    python scripts/scene_inference_bench.py [--cases sym50_bs1,sym50_bs32,mixed12_bs16] [--repeat 1] [--dump-outputs DIR]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from common import card

ENC_GFLOP, PAIR_GFLOP = 1046.1 / 2, 437.3 + 373.4
CASES = dict(sym50_bs1=(50, 0, 1), sym50_bs32=(50, 0, 32), mixed12_bs16=(6, 6, 16))   # landscape views, portrait views, batch


def views(n_land, n_port, seed=21):
    from dust3r_b200.utils.synth import synth_images
    out = []
    for k in range(n_land + n_port):
        h, w = (384, 512) if k < n_land else (512, 384)
        v = synth_images(1, h, w, seed=seed + k)[0]
        out.append(dict(v, img=v['img'].pin_memory(), idx=k, instance=str(k)))
    return out


class EncoderCounter:
    """Counts the images every encode call of the library encodes (every forward runs through `_PackedModel.encode`)."""

    def __init__(self):
        from dust3r_b200.model import _PackedModel
        self.n = 0
        encode = _PackedModel.encode

        def counted(packed, imgs):
            self.n += int(imgs.shape[0])
            return encode(packed, imgs)
        _PackedModel.encode = counted


def sample(out):
    """A fixed sample of the result: every pair's pointmaps and confidences at a 7-pixel stride."""
    res = {}
    for which, key in (('pred1', 'pts3d'), ('pred1', 'conf'), ('pred2', 'pts3d_in_other_view'), ('pred2', 'conf')):
        t = out[which][key]
        items = t if isinstance(t, list) else list(t)
        res[f'{which}_{key}'] = np.concatenate([np.asarray(x.cpu())[::7, ::7].reshape(-1) for x in items])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cases', default=','.join(CASES))
    ap.add_argument('--repeat', type=int, default=1)
    ap.add_argument('--dump-outputs', default=None)
    args = ap.parse_args()
    from bench import build_model
    from dust3r_b200.image_pairs import make_pairs
    from dust3r_b200.inference import inference
    dev = torch.device('cuda:0')
    net, _ = build_model(dev)
    counter = EncoderCounter()
    for name in args.cases.split(','):
        n_land, n_port, bs = CASES[name]
        pairs = make_pairs(views(n_land, n_port), scene_graph='complete', prefilter=None, symmetrize=True)
        out = inference(pairs[:64] if n_port == 0 else pairs, net, dev, batch_size=bs, verbose=False)   # warm-up, both sizes
        torch.cuda.synchronize()
        times = []
        for _ in range(args.repeat):
            counter.n = 0
            del out
            t0 = time.perf_counter()
            out = inference(pairs, net, dev, batch_size=bs, verbose=False)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        t = float(np.median(times))
        passes = counter.n
        tflop = (passes * ENC_GFLOP + len(pairs) * PAIR_GFLOP) / 1e3
        print(json.dumps(dict(case=name, views=n_land + n_port, pairs=len(pairs), batch_size=bs, seconds=[round(x, 3) for x in times],
                              pairs_per_s=round(len(pairs) / t, 1), encoder_passes=passes, algorithmic_tflop=round(tflop, 1),
                              algorithmic_tflop_per_s=round(tflop / t, 1), card=card(dev))), flush=True)
        if args.dump_outputs:
            os.makedirs(args.dump_outputs, exist_ok=True)
            np.savez(os.path.join(args.dump_outputs, f'{name}.npz'), **sample(out))
        del out


if __name__ == '__main__':
    main()
