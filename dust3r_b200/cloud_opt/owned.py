"""Scenes built from the rows of distributed.inference_sharded(keep='owned'): each rank of the group holds only the rows its
images need -- the whole row of every pair whose first image it owns, the view-2 half of every pair whose second image it
owns (distributed.PairOutputRoute).  The alignment loop and the differentiable objective need nothing else (the engine packs
its own images' entries); what needs more is assembled here with collectives on the scene's device:

  share_im_conf      each owner forms its images' confidence maxima from its own entries; one broadcast per owner.
  edge_scores        the spanning tree's edge scores, each computed on the rank keeping the whole row; one all-reduce.
  kept_rows          pred_i / pred_j / conf_i / conf_j as the spanning-tree walk reads them: a row this rank does not keep
                     is broadcast from its keeper when the walk first reads it.  Every rank runs the same walk, which
                     reads rows in an order fixed by the scores and the graph, so every rank issues the same broadcasts.
  share_edge_rows    rows of a per-edge parameter computed on the rank keeping each edge; one broadcast per keeper.
  share_image_rows   the depth map of every image, computed on its owner; one broadcast per image."""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

from .commons import edge_conf, edge_str


def shard_of(scene):
    """The _AlignShard of a scene built from kept rows, else None."""
    shard = scene.__dict__.get('_align_shard')
    return shard if shard is not None and shard.partial else None


def _owners(scene, shard):
    owner = np.empty(scene.n_imgs, dtype=np.int64)
    for r, (a, b) in enumerate(shard.shards):
        owner[a:b] = r
    return owner


def edge_keepers(scene):
    """Rank keeping the whole row of every edge: the owner of its first image."""
    shard = shard_of(scene)
    return _owners(scene, shard)[np.asarray([i for i, j in scene.edges], dtype=np.int64)]


def keeps_edge(scene):
    """Boolean per edge: whether this rank keeps the edge's whole row."""
    shard = shard_of(scene)
    return edge_keepers(scene) == dist.get_rank(shard.group)


def owns_image(scene, img):
    shard = shard_of(scene)
    a, b = shard.shards[dist.get_rank(shard.group)]
    return a <= img < b


@torch.no_grad()
def share_im_conf(scene):
    """Every owner's images' im_conf (exact: its entries are all the entries of its images) to every rank."""
    shard = shard_of(scene)
    for r, (a, b) in enumerate(shard.shards):
        if b == a:
            continue
        flat = torch.cat([scene.im_conf[i].data.reshape(-1) for i in range(a, b)])
        dist.broadcast(flat, src=shard.src(r), group=shard.group)
        off = 0
        for i in range(a, b):
            c = scene.im_conf[i].data
            c.copy_(flat[off:off + c.numel()].view_as(c))
            off += c.numel()


@torch.no_grad()
def edge_scores(scene):
    """{(i, j): score} of every edge (commons.edge_conf), each computed by the rank keeping the whole row and combined with
    one all-reduce of E float64 values: one non-zero term per edge, so the sum is the keeper's value exactly."""
    shard = shard_of(scene)
    mine = keeps_edge(scene)
    vals = np.zeros(scene.n_edges, dtype=np.float64)
    for e, (i, j) in enumerate(scene.edges):
        if mine[e]:
            vals[e] = edge_conf(scene.conf_i, scene.conf_j, edge_str(i, j))
    t = torch.from_numpy(vals).to(scene.device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM, group=shard.group)
    return {ij: float(v) for ij, v in zip(scene.edges, t.cpu().tolist())}


class _Rows:
    """One of the four per-edge dictionaries, read by key; rows this rank does not keep come from their keeper."""

    def __init__(self, scene, name, cache):
        self.scene, self.name, self.cache = scene, name, cache
        shard = shard_of(scene)
        self.shard, self.rank = shard, dist.get_rank(shard.group)
        self.keeper = edge_keepers(scene)
        self.edge_of = {edge_str(i, j): e for e, (i, j) in enumerate(scene.edges)}

    def __getitem__(self, key):
        hit = self.cache.get((self.name, key))
        if hit is not None:
            return hit
        e = self.edge_of[key]
        i, j = self.scene.edges[e]
        r = int(self.keeper[e])
        if r == self.rank:
            t = getattr(self.scene, self.name)[key].detach().contiguous()
        else:
            hw = self.scene.imshapes[i if self.name.endswith('_i') else j]
            t = torch.empty(tuple(hw) + ((3,) if self.name.startswith('pred') else ()), device=self.scene.device)
        dist.broadcast(t, src=self.shard.src(r), group=self.shard.group)
        self.cache[(self.name, key)] = t
        return t


def kept_rows(scene):
    """(pred_i, pred_j, conf_i, conf_j) for the spanning-tree walk (see the module docstring)."""
    cache = {}
    return tuple(_Rows(scene, name, cache) for name in ('pred_i', 'pred_j', 'conf_i', 'conf_j'))


@torch.no_grad()
def share_edge_rows(scene, param):
    """Rows of a per-edge parameter (E, ...) from the rank keeping each edge to every rank, one broadcast per keeper."""
    shard = shard_of(scene)
    keeper = edge_keepers(scene)
    for r in range(len(shard.shards)):
        sel = np.flatnonzero(keeper == r)
        if len(sel) == 0:
            continue
        idx = torch.from_numpy(sel).to(param.device)
        rows = param.data.index_select(0, idx)
        dist.broadcast(rows, src=shard.src(r), group=shard.group)
        param.data.index_copy_(0, idx, rows)


@torch.no_grad()
def share_image_rows(scene):
    """Every image's (trainable) depth map from its owner to every rank, one broadcast per image."""
    shard = shard_of(scene)
    owner = _owners(scene, shard)
    for i in range(scene.n_imgs):
        row = scene.im_depthmaps[i]
        if row.requires_grad:
            dist.broadcast(row.data, src=shard.src(int(owner[i])), group=shard.group)
