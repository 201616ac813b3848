"""Warp timeline of the streaming alignment kernel (debug aid, globaltimer stamps): for one iteration in steady
state prints where the iteration's wall time goes -- PDL wait release, streaming, warp-imbalance tail, ticket,
small-parameter step phases -- as the per-phase budget DESIGN.md quotes.
Usage: python scripts/align_stream_timeline.py [n_views=8]"""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from dust3r_b200 import _lib
from dust3r_b200.cloud_opt import global_aligner
from common import card, events_ms, synth_on_device


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    dev = torch.device('cuda')
    edges = [(i, j) for i in range(n) for j in range(i)]
    out = synth_on_device(n, edges, 384, 512, dev)
    net = global_aligner(out, dev, verbose=False)
    eng = net._get_engine(); net._engine_push(eng)
    assert eng.kernel == 'stream'
    eng.run(20); torch.cuda.synchronize()
    lib = _lib.get_lib()
    nw = eng.stream_grid * 8
    rows = []
    for rep in range(5):
        buf = torch.zeros((nw + 4, 4), dtype=torch.int64, device=dev)
        lib.d3r_align_set_debug(buf.data_ptr())
        # the stamps of the LAST iteration of the batch survive; its predecessor ran right before it (steady state)
        eng.run(8, reset_adam=False); torch.cuda.synchronize()
        lib.d3r_align_set_debug(None)
        traw = buf.cpu().numpy().astype(np.float64)
        t = traw[:nw]
        st = traw[nw:].reshape(-1)[:12]
        t0 = t[:, 1].min()          # first warp released from griddepcontrol.wait
        us = lambda x: (x - t0) / 1e3
        entry, rel, done, tick = us(t[:, 0]), us(t[:, 1]), us(t[:, 2]), us(t[:, 3])
        r = dict(warps=nw, entry_min=entry.min(), entry_p50=float(np.median(entry)), release_max=rel.max(),
                 stream_done_p50=float(np.median(done)), stream_done_p05=float(np.percentile(done, 5)), stream_done_max=done.max(),
                 ticket_max=tick.max(), small_phases=[round(float(us(x)), 2) for x in st.tolist()])
        rows.append(r)
    r = rows[-1]
    print(json.dumps({k: (round(v, 2) if isinstance(v, float) else v) for k, v in r.items()}))
    ms = events_ms(lambda: eng.run(300, reset_adam=False), 1, 0)
    print(json.dumps(dict(us_per_iter=ms / 300 * 1e3, n=n, E=len(edges), card=card(dev))))


if __name__ == '__main__':
    main()
