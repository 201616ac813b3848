"""Multi-GPU data parallelism of the pairwise forward (one process per GPU, torch.distributed / NCCL).

The reference runs inference on a single device (SURVEY §2b: no collective on the inference path).  Pairs are
independent, so the pair list is split into contiguous per-rank slices (global order preserved -> pair
indexing stays bit-exact), every rank holds a replica of the weights, and ONE all-gather of the per-pair
outputs rebuilds the full `inference()` result on every rank before global alignment (BASELINE north_star;
NVLink 5 / NVSwitch: any-to-any full bandwidth, so a plain ring/NVLS all-gather is bandwidth-optimal).

The collective is a single `all_gather_into_tensor` of one packed fp32 buffer: row = one pair =
[ pts3d (H*W*3) | conf (H*W) | pts3d_in_other_view (H*W*3) | conf (H*W) ]  (6.29 MB at 512x384); the result
tensors handed to the caller are VIEWS of the gathered buffer (no unpacking copy when the pair count divides
the world size; one row gather otherwise).  `PairOutputGather` is the object both `inference_sharded` and
`bench.py --gpus N` use; with `async_op=True` it double-buffers so that the gather of step k overlaps the
forward of step k+1.  Works with backend 'nccl' (GPU) and 'gloo' (CPU tests).

Global alignment shards the other way round: `global_aligner_sharded` gives every rank a contiguous range of images
(`shard_images`); each rank streams only those images' observations and the ranks exchange the fixed-point accumulator
block with one all-reduce per iteration (cloud_opt/engine.py)."""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

from .inference import inference, check_if_same_size
from .utils.device import collate_with_cat


def shard_bounds(n_items: int, world: int, rank: int):
    """Contiguous balanced split: the first (n % world) ranks get one extra item."""
    base, extra = divmod(n_items, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def shard_images(imshapes, degrees, world):
    """Contiguous image ranges [lo, hi), one per rank, balanced by the alignment kernel's streaming cost: 64-pixel slots x
    (entries of the image + fixed per-pixel work), the cost build_stream_items balances its warps by.  Every boundary is
    the image boundary closest to an even split, so each rank's cost is within one image's cost of total / world.  With
    fewer images than ranks some ranges are empty; those ranks still take part in every collective."""
    from .cloud_opt.engine import SLOT_PX, stream_cost
    slots = [(h * w + SLOT_PX - 1) // SLOT_PX for h, w in imshapes]
    cum = np.concatenate([[0.0], np.cumsum(stream_cost(slots, degrees))])
    n, world = len(imshapes), int(world)
    bounds = [0]
    for r in range(1, world):
        target = cum[-1] * r / world
        b = int(np.searchsorted(cum, target, side='left'))      # first boundary at or past the target
        if b > 0 and target - cum[b - 1] <= cum[b] - target:    # the one before it is closer
            b -= 1
        bounds.append(min(max(b, bounds[-1]), n))
    bounds.append(n)
    return [(bounds[r], bounds[r + 1]) for r in range(world)]


class _AlignShard:
    """What a sharded scene's engine needs: the image range of every rank and the process group.  Shared, not copied, by
    deepcopy (mask_sky copies the scene; a process group cannot be copied)."""

    def __init__(self, shards, group):
        self.shards, self.group = shards, group

    def __deepcopy__(self, memo):
        return self


def global_aligner_sharded(dust3r_output, device, mode=None, group=None, **optim_kw):
    """global_aligner() whose alignment loop runs on every rank of `group` (default: the whole default group), each rank
    streaming the observations of its own contiguous range of images (shard_images) and all ranks combining the exact
    fixed-point sums with one all-reduce per iteration.  Every rank passes the same full `dust3r_output` (inference_sharded
    returns it on every rank) and ends with the same aligned scene.

    Without an initialised process group, or in a group of one rank, this is global_aligner().  PairViewer has no loop
    and is returned as global_aligner builds it.  On the returned scene compute_global_alignment (every init=), scene()
    under no_grad, the getters, clean_pointcloud and mask_sky behave as on one GPU; the differentiable objective
    (loss.backward(), ret_details=True) raises NotImplementedError.  The predictions still live whole on every rank: only
    the packed observations and the per-pixel Adam state are divided."""
    from .cloud_opt import GlobalAlignerMode, global_aligner
    mode = GlobalAlignerMode.PointCloudOptimizer if mode is None else mode
    scene = global_aligner(dust3r_output, device, mode=mode, **optim_kw)
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return scene
    if mode is GlobalAlignerMode.PairViewer:
        return scene
    degrees = [0] * scene.n_imgs
    for i, j in scene.edges:
        degrees[i] += 1
        degrees[j] += 1
    scene._align_shard = _AlignShard(shard_images(scene.imshapes, degrees, dist.get_world_size(group)), group)
    return scene


class PairOutputGather:
    """One packed send buffer + `depth` gathered buffers for a fixed problem shape.

    n_pairs: GLOBAL number of pairs; hw1 / hw2: (H, W) of the first / second view's predictions; has_conf:
    whether the head produces confidences (conf_mode is not None).  `gather(pred1, pred2)` packs this rank's
    rows with one copy per tensor straight into the send buffer and issues the single collective."""

    def __init__(self, n_pairs, hw1, hw2, has_conf, device, group=None, depth=1):
        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.n_pairs = int(n_pairs)
        self.counts = [shard_bounds(n_pairs, self.world, r)[1] - shard_bounds(n_pairs, self.world, r)[0] for r in range(self.world)]
        self.rows = max(self.counts)                       # rows every rank contributes (padded)
        self.hw1, self.hw2, self.has_conf = tuple(hw1), tuple(hw2), bool(has_conf)
        a1, a2 = hw1[0] * hw1[1], hw2[0] * hw2[1]
        c = 1 if has_conf else 0
        self.cols = [('pred1', 'pts3d', 3 * a1, tuple(hw1) + (3,)), ('pred1', 'conf', c * a1, tuple(hw1)),
                     ('pred2', 'pts3d_in_other_view', 3 * a2, tuple(hw2) + (3,)), ('pred2', 'conf', c * a2, tuple(hw2))]
        self.width = sum(w for _, _, w, _ in self.cols)
        self.device = torch.device(device)
        self.send = [torch.zeros((self.rows, self.width), dtype=torch.float32, device=self.device) for _ in range(depth)]
        self.recv = [torch.empty((self.world * self.rows, self.width), dtype=torch.float32, device=self.device) for _ in range(depth)]
        self.work = [None] * depth
        self.k = 0
        self.even = all(cnt == self.rows for cnt in self.counts)
        if not self.even:
            idx = [r * self.rows + j for r in range(self.world) for j in range(self.counts[r])]
            self._row_index = torch.tensor(idx, dtype=torch.long, device=self.device)

    @property
    def bytes_per_rank(self):
        return self.rows * self.width * 4

    def gather(self, pred1, pred2, async_op=False):
        """pred1 / pred2: this rank's prediction dicts (None for a rank without pairs).  Returns the slot index;
        `result(slot)` waits (if asynchronous) and returns the full-result dicts."""
        k = self.k % len(self.send)
        self.k += 1
        if self.work[k] is not None:
            self.work[k].wait()
            self.work[k] = None
        send = self.send[k]
        preds = dict(pred1=pred1, pred2=pred2)
        off = 0
        for which, key, w, _ in self.cols:
            if w and preds[which] is not None:
                # the packed model's forward names view 2's pointmap 'pts3d' until model.forward() renames it (model.py:199-211)
                t = preds[which][key] if key in preds[which] else preds[which]['pts3d']
                send[:t.shape[0], off:off + w].copy_(t.reshape(t.shape[0], w), non_blocking=True)
            off += w
        # ---- the one collective of the path ----
        self.work[k] = dist.all_gather_into_tensor(self.recv[k], send, group=self.group, async_op=async_op)
        return k

    def wait(self, k=None):
        for j in (range(len(self.work)) if k is None else [k]):
            if self.work[j] is not None:
                self.work[j].wait()
                self.work[j] = None

    def result(self, k):
        self.wait(k)
        full = self.recv[k] if self.even else self.recv[k].index_select(0, self._row_index)
        out = dict(pred1={}, pred2={})
        off = 0
        for which, key, w, shape in self.cols:
            if w:
                out[which][key] = full[:, off:off + w].unflatten(1, shape)
            off += w
        return out['pred1'], out['pred2']


@torch.no_grad()
def inference_sharded(pairs, model, device, batch_size=8, verbose=False, group=None, gather_device=None, return_images=True):
    """inference() over this rank's slice of `pairs` + ONE all-gather -> the full result dict on every rank.

    Same return structure as inference(); tensors live on `gather_device` (default: CPU like the reference;
    pass the CUDA device to keep them resident for global_aligner -- they are then views of the gathered
    buffer).  All pairs must share one image size per view (what make_pairs over load_images(size=...) yields;
    mixed sizes make inference() return lists, which have no packed row layout).  return_images=False leaves the collated
    'img' tensors out of view1 / view2 (2.4 MB per view and pair at 512x384 of pure host copying; the aligner only uses them
    for colours)."""
    if not (dist.is_available() and dist.is_initialized()):
        return inference(pairs, model, device, batch_size=batch_size, verbose=verbose)
    if len(pairs) == 0:
        raise ValueError('inference_sharded: empty pair list')
    if not check_if_same_size(pairs):
        raise ValueError('inference_sharded needs all pairs to share one image size per view (run mixed-size pair lists through inference())')
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    lo, hi = shard_bounds(len(pairs), world, rank)
    local = inference(pairs[lo:hi], model, device, batch_size=batch_size, verbose=verbose, keep_on_device=True,
                      return_images=False) if hi > lo else None
    backend = dist.get_backend(group)
    comm_dev = torch.device(device) if backend == 'nccl' else torch.device('cpu')
    # shapes come from each view's own images, so a rank without pairs builds the same row layout as the others
    hw1 = tuple(int(s) for s in pairs[0][0]['img'].shape[-2:])
    hw2 = tuple(int(s) for s in pairs[0][1]['img'].shape[-2:])
    has_conf = _has_conf(model, local)
    g = PairOutputGather(len(pairs), hw1, hw2, has_conf, comm_dev, group=group)
    k = g.gather(local['pred1'] if local else None, local['pred2'] if local else None)
    p1, p2 = g.result(k)
    out_dev = torch.device('cpu') if gather_device is None else torch.device(gather_device)
    if out_dev != comm_dev:
        p1 = {key: v.to(out_dev) for key, v in p1.items()}
        p2 = {key: v.to(out_dev) for key, v in p2.items()}
    # the views (images, indices) are inputs every rank already holds: rebuild them locally in global order
    drop = (lambda v: v) if return_images else (lambda v: {k: x for k, x in v.items() if k != 'img'})
    view1 = collate_with_cat([drop(a) for a, b in pairs])
    view2 = collate_with_cat([drop(b) for a, b in pairs])
    return dict(view1=view1, view2=view2, pred1=p1, pred2=p2, loss=None)


def _has_conf(model, local):
    """Every rank must agree on the row layout: the model's head decides (conf_mode None -> no 'conf' key)."""
    if hasattr(model, 'conf_mode'):
        return model.conf_mode is not None
    if local is not None:
        return 'conf' in local['pred1']
    return True
