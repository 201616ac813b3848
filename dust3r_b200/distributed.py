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

A pair list of several image sizes (portrait and landscape photos) has no fixed row width: `MixedPairOutputGather` packs
every rank's rows, each of its own pair's size, back to back into one send buffer padded to the largest rank's, and the
same single all-gather rebuilds inference()'s per-pair lists as views of the gathered buffer.

Global alignment shards the other way round: `global_aligner_sharded` gives every rank a contiguous range of images
(`shard_images`); each rank streams only those images' observations and the ranks exchange the fixed-point accumulator
block with one all-reduce per iteration (cloud_opt/engine.py).

`inference_sharded(..., keep='owned')` replaces the all-gather by ONE `all_to_all_single` (`PairOutputRoute`): the image
ranges are decided from the pair list before the forward, and each rank ends up holding only the rows its images need --
the whole row of every pair whose first image it owns, the view-2 half of every pair whose second image it owns -- so that
neither the forward output nor the observations of a scene have to fit on one GPU."""
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
    """What a sharded scene's engine needs: the image range of every rank and the process group; `partial` when the scene
    holds only the rows of inference_sharded(keep='owned').  Shared, not copied, by deepcopy (mask_sky copies the scene; a
    process group cannot be copied)."""

    def __init__(self, shards, group, partial=False):
        self.shards, self.group, self.partial = shards, group, partial

    def __deepcopy__(self, memo):
        return self

    def owner(self, img):
        """Rank of the group whose image range holds image `img`."""
        return next(r for r, (a, b) in enumerate(self.shards) if a <= img < b)

    def src(self, r):
        """Global rank of rank r of the group (what the collectives take as src)."""
        return dist.get_global_rank(self.group, r) if self.group is not None else r


class OwnedRows:
    """The extra entry ('owned') of an inference_sharded(keep='owned') result: the image range of every rank (shard_images),
    the size of the group they were cut for, every image's (H, W), and the bytes of each buffer the routing allocated on
    this rank, as (name, device type, bytes)."""

    def __init__(self, shards, world, imshapes, allocated=()):
        self.shards, self.world = [tuple(s) for s in shards], int(world)
        self.imshapes = [tuple(s) for s in imshapes]
        self.allocated = list(allocated)


def global_aligner_sharded(dust3r_output, device, mode=None, group=None, **optim_kw):
    """global_aligner() whose alignment loop runs on every rank of `group` (default: the whole default group), each rank
    streaming the observations of its own contiguous range of images (shard_images) and all ranks combining the exact
    fixed-point sums with one all-reduce per iteration.  Every rank passes its own `dust3r_output` and ends with the same
    aligned scene.

    `dust3r_output` is either the full result (inference_sharded(keep='all') returns it on every rank) or the rows this
    rank keeps (inference_sharded(keep='owned')): the scene then holds only those rows, takes the image ranges from the
    output's 'owned' entry (ValueError when they were cut for a group of another size), assembles im_conf with one
    broadcast per owner, and runs init='mst' / 'known_poses' with the per-edge work on the rank that keeps the edge
    (cloud_opt/owned.py).  PairViewer needs every pair and is refused for such an output.

    Without an initialised process group, or in a group of one rank, this is global_aligner().  PairViewer has no loop
    and is returned as global_aligner builds it.  On the returned scene compute_global_alignment (every init=), scene(),
    the getters, clean_pointcloud and mask_sky behave as on one GPU, and so does the differentiable objective:
    `loss = scene(); loss.backward()` fills every trainable parameter's .grad and ModularPointCloudOptimizer's
    scene(ret_details=True) returns the per-edge losses.  scene() is a collective, as compute_global_alignment is: every
    rank of the group calls it, it evaluates at rank 0's parameters, and every rank gets the same loss, details and .grad
    (each rank's pixel pass covers its own images; one all-reduce of the sums, then one broadcast per owner of its images'
    log-depth gradients).  With the full result every rank holds all the predictions and only the packed observations and
    the per-pixel Adam state are divided; with the owned rows the predictions are divided too."""
    from .cloud_opt import GlobalAlignerMode, global_aligner
    mode = GlobalAlignerMode.PointCloudOptimizer if mode is None else mode
    owned = dust3r_output.get('owned') if isinstance(dust3r_output, dict) else None
    if owned is not None:
        return _owned_scene(dust3r_output, owned, device, mode, group, optim_kw)
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


def _owned_scene(out, owned, device, mode, group, optim_kw):
    """global_aligner_sharded over the rows of inference_sharded(keep='owned')."""
    from .cloud_opt import GlobalAlignerMode
    from .cloud_opt.owned import share_im_conf
    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    if owned.world != world:
        raise ValueError(f'this output keeps the rows of a group of {owned.world} ranks; the alignment group has {world}: '
                         'run inference_sharded and global_aligner_sharded over the same group')
    if mode is GlobalAlignerMode.PairViewer:
        raise ValueError("PairViewer needs the predictions of every pair: run inference_sharded(keep='all') for it")
    optim_kw.pop('early_upload', None)      # the kept rows already live where inference_sharded put them
    scene = mode.optimizer_class(out['view1'], out['view2'], out['pred1'], out['pred2'], imshapes=owned.imshapes, **optim_kw)
    scene = scene.to(device, non_blocking=True)
    if world > 1:       # in a group of one the rank keeps every row: the scene is global_aligner's
        scene._align_shard = _AlignShard(owned.shards, group, partial=True)
        share_im_conf(scene)
    return scene


def pair_graph(pairs):
    """(edges, imshapes) of a make_pairs list: (i, j) of every pair from view['idx'], and (H, W) of every image from its
    view's tensor.  Image ids must be 0 .. n-1, each view must hold one image, and every image one size."""
    edges, shapes = [], {}
    for a, b in pairs:
        ij = []
        for v in (a, b):
            if int(v['img'].shape[0]) != 1:
                raise ValueError("keep='owned' needs one image per view (make_pairs over load_images)")
            img = int(np.asarray(v['idx']).reshape(-1)[0])
            hw = tuple(int(s) for s in v['img'].shape[-2:])
            if shapes.setdefault(img, hw) != hw:
                raise ValueError(f'image {img} appears with two sizes')
            ij.append(img)
        edges.append(tuple(ij))
    if sorted(shapes) != list(range(len(shapes))):
        raise ValueError('image ids (view["idx"]) must be 0 .. n-1')
    return edges, [shapes[i] for i in range(len(shapes))]


class PairOutputRoute:
    """The rows of a pair list every rank keeps and the ONE all_to_all_single that takes them there.

    edges: (i, j) of every pair of the global list; imshapes: (H, W) of every image; shards: the image range of every rank
    (shard_images); has_conf: whether the head produces confidences.  Rank r computes the contiguous slice
    shard_bounds(E, world, r) of the pairs.  Of pair e = (i, j) the owner of i keeps the whole row (pts3d, conf,
    pts3d_in_other_view, conf: both pointmaps are in camera i's frame, so every edge is complete on one rank) and the owner
    of j also keeps the view-2 half (the (e, side 1) entry its alignment engine streams); no other rank keeps anything of e.

    What rank r sends rank d is four blocks, each in pair order: view-1 pointmaps and confidences of the whole rows, view-2
    pointmaps and confidences of the whole rows and the halves.  A stacked slice output fills each block with one
    index_select, and every kept tensor is a view of the receive buffer.  Split sizes follow from the pair list alone, so
    no sizes are exchanged.  `allocated` lists (name, device type, bytes) of every buffer the route allocates."""

    def __init__(self, edges, imshapes, shards, has_conf, device, group=None):
        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if len(shards) != self.world:
            raise ValueError(f'{len(shards)} image ranges for a group of {self.world} ranks')
        self.imshapes = [tuple(int(s) for s in hw) for hw in imshapes]
        owner = np.empty(len(self.imshapes), dtype=np.int64)
        for r, (a, b) in enumerate(shards):
            owner[a:b] = r
        ei = np.asarray([i for i, j in edges], dtype=np.int64)
        ej = np.asarray([j for i, j in edges], dtype=np.int64)
        self.ei, self.ej = ei, ej
        self.own1, self.own2 = owner[ei], owner[ej]
        area = np.asarray([h * w for h, w in self.imshapes], dtype=np.int64)
        self.area = (area[ei], area[ej])
        self.n_pairs = len(ei)
        self.bounds = [shard_bounds(self.n_pairs, self.world, r) for r in range(self.world)]
        self.has_conf = bool(has_conf)
        # (prediction dict, key, side, channels): side 0 = view 1 (whole rows only), side 1 = view 2 (rows and halves)
        blocks = [('pred1', 'pts3d', 0, 3), ('pred1', 'conf', 0, 1), ('pred2', 'pts3d_in_other_view', 1, 3), ('pred2', 'conf', 1, 1)]
        self.blocks = blocks if self.has_conf else [blocks[0], blocks[2]]
        self.device = torch.device(device)
        self.send_splits = [self._floats(self.rank, d) for d in range(self.world)]
        self.recv_splits = [self._floats(r, self.rank) for r in range(self.world)]
        self.allocated = []
        self.send = None

    def members(self, r, d):
        """Global ids of the pairs of rank r's slice that rank d keeps, in order: (whole rows, whole rows and halves)."""
        lo, hi = self.bounds[r]
        e = np.arange(lo, hi)
        whole = self.own1[lo:hi] == d
        return e[whole], e[whole | (self.own2[lo:hi] == d)]

    def _floats(self, r, d):
        rows = self.members(r, d)
        return int(sum(ch * self.area[side][rows[side]].sum() for _, _, side, ch in self.blocks))

    def _alloc(self, name, floats, device):
        t = torch.empty((floats,), dtype=torch.float32, device=device)
        self.allocated.append((name, t.device.type, 4 * floats))
        return t

    def pack(self, pred1, pred2):
        """Copies this rank's slice output into the send buffer, destination by destination.  pred1 / pred2: the
        prediction dicts of inference() over the slice (stacked tensors or per-pair lists), None for a rank without pairs."""
        lo, hi = self.bounds[self.rank]
        self.send = self._alloc('send', sum(self.send_splits), self.device)
        if hi == lo:
            return
        preds = dict(pred1=pred1, pred2=pred2)
        srcs = []
        for which, key, side, ch in self.blocks:
            # the packed model's forward names view 2's pointmap 'pts3d' until model.forward() renames it (model.py:199-211)
            t = preds[which][key] if key in preds[which] else preds[which]['pts3d']
            if torch.is_tensor(t):
                t = t.to(self.device, torch.float32)        # no copy unless gloo (host memory) or another dtype
            srcs.append(t)
        off = 0
        for d in range(self.world):
            rows = self.members(self.rank, d)
            for t, (_, _, side, ch) in zip(srcs, self.blocks):
                sel = rows[side]
                n = int(ch * self.area[side][sel].sum())
                block = self.send[off:off + n]
                if len(sel) == 0:
                    continue
                if torch.is_tensor(t):
                    idx = torch.from_numpy(sel - lo).to(t.device)
                    torch.index_select(t.reshape(t.shape[0], -1), 0, idx, out=block.view(len(sel), -1))
                else:
                    o = 0
                    for e in sel:
                        src = t[e - lo].reshape(-1)
                        block[o:o + src.numel()].copy_(src, non_blocking=True)
                        o += src.numel()
                off += n

    def exchange(self, out_device=None):
        """The one collective; returns (pred1, pred2) with one entry per pair of the global list: a view of the receive
        buffer (on `out_device`, default the route's device) for every row this rank keeps, None for the others."""
        recv = self._alloc('recv', sum(self.recv_splits), self.device)
        dist.all_to_all_single(recv, self.send, self.recv_splits, self.send_splits, group=self.group)
        self.send = None
        if out_device is not None and torch.device(out_device) != self.device:
            recv = recv.to(out_device)
            self.allocated.append(('kept', recv.device.type, 4 * recv.numel()))
        out = dict(pred1={}, pred2={})
        for which, key, _, _ in self.blocks:
            out[which][key] = [None] * self.n_pairs
        off = 0
        for r in range(self.world):
            rows = self.members(r, self.rank)
            for which, key, side, ch in self.blocks:
                imgs = self.ei if side == 0 else self.ej
                for e in rows[side]:
                    hw = self.imshapes[imgs[e]]
                    n = ch * hw[0] * hw[1]
                    out[which][key][e] = recv[off:off + n].view(hw + ((3,) if ch == 3 else ()))
                    off += n
        assert off == recv.numel()
        return out['pred1'], out['pred2']


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


def row_shapes(pairs):
    """((H, W) of view 1, (H, W) of view 2) of every row inference() returns for `pairs` -- one row per image of a pair's
    views, in order -- and the number of rows of every pair."""
    shapes, pair_rows = [], []
    for a, b in pairs:
        k = int(a['img'].shape[0])
        hw = tuple(tuple(int(s) for s in v['img'].shape[-2:]) for v in (a, b))
        shapes += [hw] * k
        pair_rows.append(k)
    return shapes, pair_rows


class MixedPairOutputGather:
    """The one all-gather of a pair list of several image sizes, whose rows have no common width.

    shapes / pair_rows: what row_shapes returns for the global list; has_conf: as for PairOutputGather.  Rank r computes the
    pairs shard_bounds(len(pair_rows), world, r).  A row is [pts3d | conf | pts3d_in_other_view | conf], each at its own
    view's size.  Every rank packs its rows back to back into one fp32 send buffer padded to the largest rank's float count,
    so rank r's rows start at r * width in the gathered buffer.  Row sizes follow from the pair list alone: every rank
    computes every rank's count, and no sizes are exchanged."""

    def __init__(self, shapes, pair_rows, has_conf, device, group=None):
        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.shapes = [(tuple(a), tuple(b)) for a, b in shapes]
        c = 1 if has_conf else 0
        # (prediction dict, key, channels, side): side 0 = view 1, side 1 = view 2; no conf column without confidences
        self.cols = [col for col in (('pred1', 'pts3d', 3, 0), ('pred1', 'conf', c, 0),
                                     ('pred2', 'pts3d_in_other_view', 3, 1), ('pred2', 'conf', c, 1)) if col[2]]
        first = np.concatenate([[0], np.cumsum(pair_rows, dtype=np.int64)])
        self.rows = [(int(first[lo]), int(first[hi])) for lo, hi in
                     (shard_bounds(len(pair_rows), self.world, r) for r in range(self.world))]
        self.start, self.counts = [], []        # every row's first float within its rank's block; every rank's floats
        for lo, hi in self.rows:
            ends = np.cumsum([0] + [self._floats(e) for e in range(lo, hi)], dtype=np.int64)
            self.start += ends[:-1].tolist()
            self.counts.append(int(ends[-1]))
        self.width = max(self.counts)
        self.device = torch.device(device)
        self.send = None

    def _layout(self, e):
        """(prediction dict, key, first float within the row, shape) of every tensor of row e."""
        out, o = [], 0
        for which, key, ch, side in self.cols:
            hw = self.shapes[e][side]
            out.append((which, key, o, hw + ((3,) if ch == 3 else ())))
            o += ch * hw[0] * hw[1]
        return out

    def _floats(self, e):
        return sum(ch * self.shapes[e][side][0] * self.shapes[e][side][1] for _, _, ch, side in self.cols)

    def pack(self, pred1, pred2):
        """Copies this rank's rows into the send buffer, one copy per tensor.  pred1 / pred2: the prediction dicts of
        inference() over this rank's pairs (stacked tensors when they share one size, per-row lists otherwise), None for a
        rank without pairs."""
        lo, hi = self.rows[self.rank]
        self.send = torch.empty((self.width,), dtype=torch.float32, device=self.device)
        self.send[self.counts[self.rank]:].zero_()
        if hi == lo:
            return
        preds = dict(pred1=pred1, pred2=pred2)
        layout = [self._layout(e) for e in range(lo, hi)]
        for k, (which, key, _, _) in enumerate(self.cols):
            # the packed model's forward names view 2's pointmap 'pts3d' until model.forward() renames it (model.py:199-211)
            t = preds[which][key] if key in preds[which] else preds[which]['pts3d']
            if torch.is_tensor(t):      # the rank's rows share one size: one strided copy into every row
                n, o, shape = hi - lo, layout[0][k][2], layout[0][k][3]
                size = int(np.prod(shape))
                rows = self.send[:self.counts[self.rank]].view(n, -1)
                rows[:, o:o + size].copy_(t.reshape(n, size), non_blocking=True)
            else:
                for e in range(lo, hi):
                    o = self.start[e] + layout[e - lo][k][2]
                    src = t[e - lo].reshape(-1)
                    self.send[o:o + src.numel()].copy_(src, non_blocking=True)

    def gather(self, out_device=None):
        """The one collective; returns (pred1, pred2) with one list entry per row of the global list, each a view of the
        gathered buffer (moved once to `out_device` when that is another device than the collective's)."""
        recv = torch.empty((self.world * self.width,), dtype=torch.float32, device=self.device)
        dist.all_gather_into_tensor(recv, self.send, group=self.group)
        self.send = None
        if out_device is not None and torch.device(out_device) != self.device:
            recv = recv.to(out_device)
        out = dict(pred1={}, pred2={})
        for which, key, _, _ in self.cols:
            out[which][key] = []
        for r, (lo, hi) in enumerate(self.rows):
            for e in range(lo, hi):
                base = r * self.width + self.start[e]
                for which, key, o, shape in self._layout(e):
                    out[which][key].append(recv[base + o:base + o + int(np.prod(shape))].view(shape))
        return out['pred1'], out['pred2']


@torch.no_grad()
def inference_sharded(pairs, model, device, batch_size=8, verbose=False, group=None, gather_device=None, return_images=True,
                      keep='all'):
    """inference() over this rank's slice of `pairs` + ONE collective.

    keep='all': one all-gather -> the full result dict on every rank.  Same return structure as inference() (lists with one
    entry per pair when the list holds several image sizes, MixedPairOutputGather); tensors live on `gather_device`
    (default: CPU like the reference; pass the CUDA device to keep them resident for global_aligner -- they are then views
    of the gathered buffer).

    keep='owned': the image ranges of global_aligner_sharded (shard_images over the pair graph) are decided before the
    forward, and one all_to_all_single (PairOutputRoute) leaves each rank holding only the rows its images need.  pred1 /
    pred2 then hold one entry per pair: the kept tensor (on `gather_device`) or None, and the extra entry 'owned'
    (OwnedRows) carries the image ranges and the group size for global_aligner_sharded.  Per rank, device memory peaks at
    its slice's output, one reordered copy of it (NCCL; gloo sends from host memory) and the rows it keeps.

    return_images=False leaves the collated 'img' tensors out of view1 / view2 (2.4 MB per view and pair at 512x384 of pure
    host copying; the aligner only uses them for colours)."""
    if keep not in ('all', 'owned'):
        raise ValueError(f"keep must be 'all' or 'owned', not {keep!r}")
    if not (dist.is_available() and dist.is_initialized()):
        return inference(pairs, model, device, batch_size=batch_size, verbose=verbose)
    if len(pairs) == 0:
        raise ValueError('inference_sharded: empty pair list')
    # decided from the whole list, as inference() decides it: a rank whose own slice is uniform still returns lists
    mixed = not check_if_same_size(pairs)
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if keep == 'owned':
        edges, imshapes = pair_graph(pairs)
        degrees = np.bincount(np.asarray(edges).reshape(-1), minlength=len(imshapes)).tolist()
        shards = shard_images(imshapes, degrees, world)
    lo, hi = shard_bounds(len(pairs), world, rank)
    local = inference(pairs[lo:hi], model, device, batch_size=batch_size, verbose=verbose, keep_on_device=True,
                      return_images=False) if hi > lo else None
    backend = dist.get_backend(group)
    comm_dev = torch.device(device) if backend == 'nccl' else torch.device('cpu')
    drop = (lambda v: v) if return_images else (lambda v: {k: x for k, x in v.items() if k != 'img'})
    if keep == 'owned':
        route = PairOutputRoute(edges, imshapes, shards, _has_conf(model, local), comm_dev, group=group)
        route.pack(local['pred1'] if local else None, local['pred2'] if local else None)
        del local       # the slice output is not needed once it sits in the send buffer
        out_dev = torch.device('cpu') if gather_device is None else torch.device(gather_device)
        p1, p2 = route.exchange(out_dev)
        view1 = collate_with_cat([drop(a) for a, b in pairs], lists=mixed)
        view2 = collate_with_cat([drop(b) for a, b in pairs], lists=mixed)
        return dict(view1=view1, view2=view2, pred1=p1, pred2=p2, loss=None,
                    owned=OwnedRows(shards, world, imshapes, route.allocated))
    if mixed:
        shapes, pair_rows = row_shapes(pairs)
        g = MixedPairOutputGather(shapes, pair_rows, _has_conf(model, local), comm_dev, group=group)
        g.pack(local['pred1'] if local else None, local['pred2'] if local else None)
        del local       # the slice output is not needed once it sits in the send buffer
        p1, p2 = g.gather(torch.device('cpu') if gather_device is None else torch.device(gather_device))
        view1 = collate_with_cat([drop(a) for a, b in pairs], lists=True)
        view2 = collate_with_cat([drop(b) for a, b in pairs], lists=True)
        return dict(view1=view1, view2=view2, pred1=p1, pred2=p2, loss=None)
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
