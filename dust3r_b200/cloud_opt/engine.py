"""Host driver of the fused alignment kernels (csrc/align_stream.cu when every image has P % 4 == 0, csrc/align_step.cu
for any shape) — builds the HBM layout the kernels stream and launches `d3r_align_run` through the C ABI.

HBM layout (all fp32, owned by torch):
  obs        float4[ sum over entries P_img ]   (pred.x, pred.y, pred.z, conf_trf(conf)) per pixel;
             entry = (edge, side); entries of one image are contiguous in a CSR so a CTA walks them
             while its pixels' world points stay in registers.  32*E*P bytes, read once / iteration.
  logd       float[ sum_i stride_i ]            log-depth (+ exp_avg, exp_avg_sq): 24*n*P bytes r+w.
  small      float[ 7n + 2n + 2n + 8E + 2E ]    poses / focals / pp / pairwise poses / adaptors.

Sharded over the ranks of a process group (`shards=`), each rank packs and streams only its own images' entries and runs
every iteration as pixel pass -> one all-reduce of the fixed-point accumulator block -> small step (d3r_align_pixel_pass /
d3r_align_small_step), so that every rank computes the same small parameters; `logd` keeps its global layout.  The
objective's gradient is split the same way (sharded_loss_and_grad: d3r_align_grad_pixel_pass -> the all-reduce ->
d3r_align_grad_small_step, then one broadcast per owner of its images' log-depth gradients).
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import List, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as tdist

from .. import _lib
from .commons import cosine_schedule, linear_schedule


_CONF_MODES = {'id': 0, 'none': 0, 'log': 1, 'sqrt': 2, 'm1': 3}

PACK_ENTRY = np.dtype([('pts', np.uint64), ('conf', np.uint64), ('obs_off', np.int64), ('area', np.int32), ('coef', np.float32)])
ITEM = np.dtype([('img', np.int32), ('slot0', np.int32), ('nslots', np.int32), ('npx', np.int32),
                 ('e0', np.int32), ('deg', np.int32), ('W', np.int32), ('u0', np.int32),
                 ('v0', np.int32), ('inv_w', np.float32), ('pix0', np.int64), ('obs0', np.int64),
                 ('slab_units', np.int32), ('reserved', np.int32)])
SLOT_PX = 64          # pixels per slot of the streaming layout (32 pixel pairs)
PIXEL_COST = 3        # streaming cost of a slot = entries of its image + PIXEL_COST (unprojection, depth Adam, item set-up)


def stream_cost(slots, degrees):
    """Streaming cost of every image (or slot): slots x (entries of the image + fixed per-pixel work)."""
    return np.asarray(slots, dtype=np.float64) * (np.asarray(degrees, dtype=np.float64) + PIXEL_COST)


def build_stream_items(imshapes, pix_off, ent_ptr, ent_obs_off, slots, ppt, warps_per_cta, max_ctas):
    """Work items of the streaming kernel (csrc/align_stream.cu).  Every image's range of 64-pixel slots is cut into
    items of <= ppt slots; the global slot sequence is split into one contiguous run per persistent warp, balanced by
    cost = slots x (entries of the image + fixed per-pixel work).  Returns (items[ITEM], warp_item_ptr[int32], ctas).
    Vectorised: ~8000 items for 8 images at 512x384 are built in about a millisecond (the item-by-item Python loop
    this replaces took longer than 300 iterations of the kernel it feeds)."""
    n = len(imshapes)
    areas = np.asarray([h * w for h, w in imshapes], dtype=np.int64)
    widths = np.asarray([w for h, w in imshapes], dtype=np.int64)
    slots = np.asarray(slots, dtype=np.int64)
    deg = np.diff(ent_ptr).astype(np.int64)
    img_first = np.concatenate([[0], np.cumsum(slots)])            # first global slot of every image
    total = int(img_first[-1])
    slot_img = np.repeat(np.arange(n), slots)                      # image of every slot, global slot order
    cost = stream_cost(1, deg[slot_img])
    cum = np.concatenate([[0.0], np.cumsum(cost)])
    n_warps = int(min(max_ctas * warps_per_cta, total))
    grid = (n_warps + warps_per_cta - 1) // warps_per_cta
    bounds = np.searchsorted(cum, cum[-1] * np.arange(n_warps + 1) / n_warps, side='left')
    bounds = np.concatenate([np.minimum(bounds, total), np.full(grid * warps_per_cta - n_warps, total, dtype=bounds.dtype)])
    bounds[0], bounds[n_warps:] = 0, total
    # segments: maximal slot ranges inside one warp's run and one image, each cut into items of <= ppt slots
    cuts = np.unique(np.concatenate([bounds, img_first]))
    seg_a, seg_b = cuts[:-1], cuts[1:]
    n_chunks = (seg_b - seg_a + ppt - 1) // ppt
    seg_of = np.repeat(np.arange(len(seg_a)), n_chunks)
    k_in = np.arange(int(n_chunks.sum())) - np.repeat(np.cumsum(n_chunks) - n_chunks, n_chunks)
    start = seg_a[seg_of] + k_in * ppt                             # first global slot of every item
    ns = np.minimum(ppt, seg_b[seg_of] - start)
    img = slot_img[start]
    s0 = start - img_first[img]                                    # slot index inside the image
    p0 = s0 * SLOT_PX
    W = widths[img]
    first_entry = np.asarray(ent_ptr, dtype=np.int64)[img]
    obs0 = np.where(deg[img] > 0, np.asarray(ent_obs_off, dtype=np.int64)[np.minimum(first_entry, len(ent_obs_off) - 1)] + p0, 0)
    arr = np.zeros(len(start), dtype=ITEM)
    arr['img'], arr['slot0'], arr['nslots'] = img, s0, ns
    arr['npx'] = np.minimum(ns * SLOT_PX, areas[img] - p0)
    arr['e0'], arr['deg'], arr['W'] = first_entry, deg[img], W
    arr['u0'], arr['v0'] = p0 % W, p0 // W
    arr['inv_w'] = (1.0 / W).astype(np.float32)
    arr['pix0'] = np.asarray(pix_off, dtype=np.int64)[img] + p0
    arr['obs0'] = obs0
    arr['slab_units'] = slots[img] * SLOT_PX
    warp_ptr = np.searchsorted(start, bounds, side='left').astype(np.int32)
    return arr, warp_ptr, grid


class AlignEngine:
    """pred_i / pred_j: per-edge (H, W, 3) pointmaps; conf_i / conf_j: per-edge RAW confidences (H, W) -- the
    confidence transform `conf_mode` (commons.py:73-80) is applied by the packing kernel.  Tensors already on
    `device` (e.g. views of inference(keep_on_device=True) / all-gather output) are read in place; everything is
    packed by ONE launch (d3r_align_pack_entries).

    shards: optional list of contiguous image ranges [lo, hi), one per rank of `group` (distributed.shard_images); this
    rank packs and streams only the entries of its own range, and run() / evaluate_loss() / sharded_loss_and_grad()
    exchange the accumulators with one all-reduce per iteration.  Streaming kernel only.  The inputs of entries outside the
    range are never read and may be None (a scene of the rows inference_sharded(keep='owned') kept)."""

    def __init__(self, edges: Sequence[Tuple[int, int]], imshapes: Sequence[Tuple[int, int]],
                 pred_i: Sequence[torch.Tensor], pred_j: Sequence[torch.Tensor],
                 conf_i: Sequence[torch.Tensor], conf_j: Sequence[torch.Tensor],
                 device, conf_mode='log', dist='l1', variant='stacked', pix_stride=None,
                 base_scale=0.5, pw_break=20.0, focal_break=20.0, kernel='auto', reverse_odd='auto', shards=None, group=None):
        self.device = _lib.require_cuda_device(device)
        self.lib = _lib.get_lib()
        self.edges = [(int(i), int(j)) for i, j in edges]
        self.imshapes = [tuple(map(int, s)) for s in imshapes]
        self.n, self.E = len(self.imshapes), len(self.edges)
        n, E = self.n, self.E
        assert dist in ('l1', 'l2')
        if conf_mode not in _CONF_MODES:
            raise ValueError(f'bad mode for {conf_mode=}')
        self.dist, self.variant = dist, variant
        self.base_scale, self.pw_break, self.focal_break = float(base_scale), float(pw_break), float(focal_break)
        areas = [h * w for h, w in self.imshapes]
        self.areas = areas
        # pixel storage stride per image (PointCloudOptimizer pads every image to max_area,
        # optimizer.py:37-45; the modular variant packs tightly)
        self.pix_stride = [int(pix_stride)] * n if pix_stride is not None else areas
        pix_off = np.zeros(n + 1, dtype=np.int64)
        pix_off[1:] = np.cumsum(self.pix_stride)
        self.pix_off = pix_off
        # streaming kernel (csrc/align_stream.cu): needs 16-byte aligned log-depth slices.  DUSt3R images are multiples
        # of the 16-pixel patch, so this is the path real inputs take; odd shapes run the general kernel.
        eligible = all(a % 4 == 0 for a in areas) and all(int(o) % 4 == 0 for o in pix_off)
        if kernel == 'auto':
            kernel = 'stream' if eligible else 'general'
        if kernel == 'stream' and not eligible:
            raise ValueError('the streaming alignment kernel needs H*W and the pixel stride of every image to be multiples of 4')
        assert kernel in ('stream', 'general')
        self.kernel = kernel
        stream = kernel == 'stream'
        self.group, self.shards = group, None
        lo, hi = 0, n
        if shards is not None:
            if not stream:
                raise ValueError('the sharded alignment runs on the streaming kernel only (every image needs H*W and its pixel '
                                 'stride to be multiples of 4)')
            self.shards = [(int(a), int(b)) for a, b in shards]
            if len(self.shards) != tdist.get_world_size(group):
                raise ValueError(f'{len(self.shards)} image ranges for a group of {tdist.get_world_size(group)} ranks')
            lo, hi = self.shards[tdist.get_rank(group)]
        self.owned = (lo, hi)
        if reverse_odd == 'auto':     # D3R_ALIGN_REVERSE=0: every iteration walks the items in the same order (A/B switch)
            reverse_odd = os.environ.get('D3R_ALIGN_REVERSE', '1') != '0'
        self.reverse_odd = bool(reverse_odd)
        chunk = self._pick_chunk_px(areas)
        self.chunk_px = chunk
        nchunks = [(a + chunk - 1) // chunk for a in areas]
        chunk_ptr = np.zeros(n + 1, dtype=np.int32)
        chunk_ptr[1:] = np.cumsum(nchunks)
        chunk_img = np.repeat(np.arange(n, dtype=np.int32), nchunks)
        # CSR image -> entries.  entry id order: for each image, incident (edge, side) sorted by edge
        ent_lists = [[] for _ in range(n)]
        for e, (i, j) in enumerate(self.edges):
            ent_lists[i].append((e, 0))
            ent_lists[j].append((e, 1))
        ent_ptr = np.zeros(n + 1, dtype=np.int32)
        ent_ptr[1:] = np.cumsum([len(l) for l in ent_lists])
        ent_edge = np.zeros(2 * E, dtype=np.int32)
        ent_obs_off = np.zeros(2 * E, dtype=np.int64)
        ent_coef = np.zeros(2 * E, dtype=np.float32)
        edge_ent = np.zeros((E, 2), dtype=np.int32)
        if variant == 'stacked':     # optimizer.py:59-60,198-199: sum / total_area per side
            tot = [sum(areas[i] for i, j in self.edges), sum(areas[j] for i, j in self.edges)]
        slots = [(a + SLOT_PX - 1) // SLOT_PX for a in areas]
        k = 0
        off = 0
        table = np.zeros(2 * E, dtype=PACK_ENTRY)
        keep = []                     # device copies of host inputs stay alive until the pack launch has run
        dev = self.device

        def on_dev(t, width):
            t = t.reshape(-1, width) if width > 1 else t.reshape(-1)
            if t.device != dev or t.dtype != torch.float32 or not t.is_contiguous():
                t = t.to(dev, torch.float32).contiguous()
                keep.append(t)
            return t
        for img in range(n):
            for (e, side) in ent_lists[img]:
                ent_edge[k] = e
                ent_obs_off[k] = off
                if variant == 'stacked':
                    ent_coef[k] = 1.0 / tot[side]
                else:                # base_opt.py:262-270: mean over pixels, then / n_edges
                    ent_coef[k] = 1.0 / (areas[img] * E)
                edge_ent[e, side] = k
                if not lo <= img < hi:      # another rank's image: its observations are not packed here
                    k += 1
                    continue
                pts, cf = (pred_i[e], conf_i[e]) if side == 0 else (pred_j[e], conf_j[e])
                if pts is None or cf is None:
                    raise ValueError(f'entry ({e}, side {side}) of image {img}, an image of this rank, was not given')
                pts, cf = on_dev(pts, 3), on_dev(cf, 1)
                assert pts.shape[0] >= areas[img] and cf.shape[0] >= areas[img]
                table[k] = (pts.data_ptr(), cf.data_ptr(), off, areas[img], ent_coef[k])
                off += slots[img] * SLOT_PX if stream else areas[img]
                k += 1
        self.total_obs = off
        self.obs_px = sum(areas[i] + areas[j] for i, j in self.edges)      # algorithmic observation count (no padding)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        self._img_hw = t(np.int32(self.imshapes))
        self._pix_off = t(pix_off)
        self._ent_ptr = t(ent_ptr)
        self._chunk_ptr = t(chunk_ptr)
        self._chunk_img = t(chunk_img)
        self._ent_edge = t(ent_edge)
        self._ent_obs_off = t(ent_obs_off)
        self._ent_coef = t(ent_coef)
        self._edge_ent = t(edge_ent)
        self.n_chunks = int(chunk_ptr[-1])
        self.max_chunks = int(max(nchunks))
        self.max_deg = int(max(len(l) for l in ent_lists))
        # observations: one launch for every entry, confidence transform and (streaming layout) loss coefficient fused
        self.obs = torch.empty((max(self.total_obs, 1), 4), dtype=torch.float32, device=dev)   # >= 1 row: a rank without images
        k0, k1 = int(ent_ptr[lo]), int(ent_ptr[hi])      # entries of the packed images (all of them unless sharded)
        table_dev = torch.from_numpy(np.ascontiguousarray(table[k0:k1]).view(np.uint8)).to(dev)
        if k1 > k0:
            _lib.launch(dev, 'd3r_align_pack_entries', table_dev.data_ptr(), k1 - k0, int(max(areas[lo:hi])), _CONF_MODES[conf_mode],
                        1 if stream else 0, self.obs.data_ptr())
        if keep:
            torch.cuda.current_stream(dev).synchronize()     # the staged copies may be freed after this point
        del keep, table_dev
        if stream:
            self._build_items(ent_ptr, ent_obs_off, [s if lo <= i < hi else 0 for i, s in enumerate(slots)])
        else:
            self._no_items()
        nws = self.lib.d3r_align_workspace_floats(n, E)
        self.workspace = torch.zeros((nws,), dtype=torch.float32, device=dev)
        if self.shards is not None:     # the int64 block [ent_acc | img_acc | overflow word] the ranks all-reduce
            off, words = C.c_int64(0), C.c_int64(0)
            _lib.check(self.lib.d3r_align_reduce_block(n, E, C.byref(off), C.byref(words)))
            self.reduce_block = (int(off.value), int(words.value))
            self._reduce = self.workspace[off.value:off.value + 2 * words.value].view(torch.int64)
        self.counters = torch.zeros((n + 2,), dtype=torch.int32, device=dev)
        self.n_small = 11 * n + 10 * E
        self.small = torch.zeros((self.n_small,), dtype=torch.float32, device=dev)
        self.small_m = torch.zeros_like(self.small)
        self.small_v = torch.zeros_like(self.small)
        self.small_trainable = torch.zeros((self.n_small,), dtype=torch.uint8, device=dev)
        self.logd = None
        self.logd_m = self.logd_v = None
        self.sched = torch.zeros((1, 4), dtype=torch.float32, device=dev)
        self.loss_out = torch.zeros((1,), dtype=torch.float32, device=dev)
        self.norm_pw_scale = True
        self.tied_focal = True

    def _call(self, fn, *args):
        """_lib.launch on the engine's device for a caller that holds the library function `fn` itself (an attribute of
        _lib.get_lib()), e.g. a test that runs a range of iterations with d3r_align_run."""
        _lib.launch(self.device, fn.__name__, *args)

    def _no_items(self):
        self.stream_grid = self.stream_ppt = self.stream_window = self.n_items = 0
        self._items = self._warp_item_ptr = self._items_rev = self._warp_item_ptr_rev = None

    def _build_items(self, ent_ptr, ent_obs_off, slots):
        """Work items over the images with slots > 0 (a sharded engine zeroes the slots of other ranks' images).  The entry
        window follows the whole graph, so that every rank's small step runs the same version."""
        lib = self.lib
        ppt = int(lib.d3r_align_stream_slots_per_item())
        wpc = int(lib.d3r_align_stream_warps_per_cta())
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        deg_max = int(np.diff(ent_ptr).max())
        window = int(min(max(deg_max, 1), lib.d3r_align_stream_max_window()))
        if sum(slots) == 0:         # a rank without images: no pixel pass, but the same small step as every other rank
            self._no_items()
            self.stream_ppt, self.stream_window = ppt, window
            return
        arr, warp_ptr, grid = build_stream_items(self.imshapes, self.pix_off, ent_ptr, ent_obs_off, slots, ppt, wpc, 2 * sms)
        assert arr.dtype.itemsize == 64 == lib.d3r_sizeof_align_item()
        dev = self.device
        self._items = torch.from_numpy(arr.view(np.uint8)).to(dev)
        self._warp_item_ptr = torch.from_numpy(warp_ptr).to(dev)
        self.n_items = len(arr)
        # reversed traversal for odd iterations: warp w walks the reverse of warp (nw-1-w)'s run, so the global streaming
        # order of an odd iteration is the exact reverse of an even one (the L2 still holds the tail of the last pass)
        self._items_rev = self._warp_item_ptr_rev = None
        if self.reverse_odd:
            arr_rev = np.ascontiguousarray(arr[::-1])
            warp_ptr_rev = (len(arr) - warp_ptr[::-1]).astype(np.int32)
            self._items_rev = torch.from_numpy(arr_rev.view(np.uint8)).to(dev)
            self._warp_item_ptr_rev = torch.from_numpy(np.ascontiguousarray(warp_ptr_rev)).to(dev)
        self.stream_grid, self.stream_ppt = grid, ppt
        self.stream_window = window

    def _pick_chunk_px(self, areas):
        """Pixels per CTA: the largest size <= the kernel's maximum for which the grid is (close to) a whole
        number of waves of 2 CTAs/SM — a ragged last wave idles most of the chip for a full CTA lifetime."""
        cmax = int(self.lib.d3r_align_chunk_pixels())
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        slots = 2 * sms
        best, best_cost = cmax, None
        for c in range(cmax, cmax // 2, -8):
            total = sum((a + c - 1) // c for a in areas)
            waves = total / slots
            cost = math.ceil(waves) / waves            # time relative to a perfectly divisible grid
            cost *= 1.0 + 0.02 * (cmax - c) / cmax      # mild preference for bigger chunks (fewer partial rows)
            if best_cost is None or cost < best_cost - 1e-9:
                best, best_cost = c, cost
        return best

    # ------------------------------------------------------------------ parameters
    def algorithmic_bytes_per_iter(self):
        """SURVEY §8d: 32*E*P (observations read once) + 24*n*P (log-depth + 2 moments r/w)."""
        return 16 * self.obs_px + 24 * sum(self.areas)

    def _offsets(self):
        n, E = self.n, self.E
        o = dict(poses=0, focals=7 * n, pp=9 * n, pw=11 * n, adapt=11 * n + 8 * E)
        return o

    def set_params(self, logd: torch.Tensor, im_poses, im_focals, im_pp, pw_poses, pw_adaptors,
                   train_poses, train_focals, train_pp, train_pw=True, train_adaptors=False,
                   norm_pw_scale=True):
        """logd: flat float32 CUDA tensor the kernel updates IN PLACE (length pix_off[-1]).
        im_focals: (n,1) tied or (n,2).  train_*: bool or per-image bool arrays."""
        n, E = self.n, self.E
        dev = self.device
        assert logd.is_cuda and logd.dtype == torch.float32 and logd.is_contiguous() and logd.numel() == int(self.pix_off[-1])
        self.logd = logd
        o = self._offsets()
        f = torch.as_tensor(im_focals, dtype=torch.float32, device=dev).reshape(n, -1)
        self.tied_focal = f.shape[1] == 1
        f2 = f.expand(n, 2) if self.tied_focal else f
        s = self.small
        s[o['poses']:o['focals']] = torch.as_tensor(im_poses, dtype=torch.float32, device=dev).reshape(-1)
        s[o['focals']:o['pp']] = f2.reshape(-1)
        s[o['pp']:o['pw']] = torch.as_tensor(im_pp, dtype=torch.float32, device=dev).reshape(-1)
        s[o['pw']:o['adapt']] = torch.as_tensor(pw_poses, dtype=torch.float32, device=dev).reshape(-1)
        s[o['adapt']:] = torch.as_tensor(pw_adaptors, dtype=torch.float32, device=dev).reshape(-1)

        def mask(flag, width):
            m = np.asarray(flag, dtype=bool)
            if m.ndim == 0:
                m = np.full((n,), bool(m))
            return np.repeat(m.astype(np.uint8)[:, None], width, axis=1).reshape(-1)
        tr = np.zeros((self.n_small,), dtype=np.uint8)
        tr[o['poses']:o['focals']] = mask(train_poses, 7)
        tr[o['focals']:o['pp']] = mask(train_focals, 2)
        tr[o['pp']:o['pw']] = mask(train_pp, 2)
        tr[o['pw']:o['adapt']] = 1 if train_pw else 0
        tr[o['adapt']:] = 1 if train_adaptors else 0
        self.small_trainable.copy_(torch.from_numpy(tr))
        self.norm_pw_scale = bool(norm_pw_scale)
        self._prepared = False

    def split_small(self, flat):
        """Views of a flat buffer in the `small` layout -- the parameters or their gradients -- one per parameter kind,
        shaped like the stacked parameters; im_focals is (n, 1) with a tied focal (both slots hold the same value)."""
        n, E = self.n, self.E
        o = self._offsets()
        f = flat[o['focals']:o['pp']].reshape(n, 2)
        return dict(im_poses=flat[o['poses']:o['focals']].reshape(n, 7),
                    im_focals=f[:, :1] if self.tied_focal else f,
                    im_pp=flat[o['pp']:o['pw']].reshape(n, 2),
                    pw_poses=flat[o['pw']:o['adapt']].reshape(E, 8),
                    pw_adaptors=flat[o['adapt']:].reshape(E, 2))

    def get_small(self):
        return {k: v.clone() for k, v in self.split_small(self.small).items()}

    def reset_adam(self):
        self.small_m.zero_()
        self.small_v.zero_()
        self.logd_m = torch.zeros_like(self.logd)
        self.logd_v = torch.zeros_like(self.logd)

    # ------------------------------------------------------------------ launches
    def _desc(self, eval_only=False):
        d = _lib.AlignDesc()
        d.n_imgs, d.n_edges, d.n_entries, d.n_chunks = self.n, self.E, 2 * self.E, self.n_chunks
        d.max_deg, d.max_chunks = self.max_deg, self.max_chunks
        d.chunk_px = self.chunk_px
        d.dist_l2 = 1 if self.dist == 'l2' else 0
        d.norm_pw_scale = int(self.norm_pw_scale)
        d.tied_focal = int(self.tied_focal)
        d.eval_only = int(eval_only)
        d.base_scale, d.pw_break, d.focal_break = self.base_scale, self.pw_break, self.focal_break
        d.adam_eps, d.beta1, d.beta2 = 1e-8, 0.9, 0.9     # base_opt.py:337
        d.img_hw = self._img_hw.data_ptr()
        d.img_pix_off = self._pix_off.data_ptr()
        d.img_ent_ptr = self._ent_ptr.data_ptr()
        d.img_chunk_ptr = self._chunk_ptr.data_ptr()
        d.chunk_img = self._chunk_img.data_ptr()
        d.ent_edge = self._ent_edge.data_ptr()
        d.ent_obs_off = self._ent_obs_off.data_ptr()
        d.ent_coef = self._ent_coef.data_ptr()
        d.edge_ent = self._edge_ent.data_ptr()
        d.obs = self.obs.data_ptr()
        d.logd = self.logd.data_ptr()
        if self.logd_m is None:
            self.reset_adam()
        d.logd_m, d.logd_v = self.logd_m.data_ptr(), self.logd_v.data_ptr()
        d.small, d.small_m, d.small_v = self.small.data_ptr(), self.small_m.data_ptr(), self.small_v.data_ptr()
        d.small_trainable = self.small_trainable.data_ptr()
        d.workspace = self.workspace.data_ptr()
        d.sched = self.sched.data_ptr()
        d.loss_out = self.loss_out.data_ptr()
        d.counters = self.counters.data_ptr()
        d.stream_kernel = 1 if self.kernel == 'stream' else 0
        d.stream_grid, d.stream_ppt, d.stream_window, d.n_items = self.stream_grid, self.stream_ppt, self.stream_window, self.n_items
        if self.n_items:
            d.items, d.warp_item_ptr = self._items.data_ptr(), self._warp_item_ptr.data_ptr()
            if self._items_rev is not None:
                d.items_rev, d.warp_item_ptr_rev = self._items_rev.data_ptr(), self._warp_item_ptr_rev.data_ptr()
        return d

    def prepare(self):
        d = self._desc()
        _lib.launch(self.device, 'd3r_align_prepare', C.byref(d))
        self._prepared = True

    @staticmethod
    def make_schedule(niter, lr, schedule='cosine', lr_min=1e-6, beta1=0.9, beta2=0.9, first_step=1):
        """Per-iteration scalars computed in double exactly as base_opt.py:352-360 + torch Adam do."""
        rows = np.zeros((max(niter, 1), 4), dtype=np.float64)
        for it in range(niter):
            t = it / niter
            if schedule == 'cosine':
                cur = cosine_schedule(t, lr, lr_min)
            elif schedule == 'linear':
                cur = linear_schedule(t, lr, lr_min)
            else:
                raise ValueError(f'bad lr {schedule=}')
            step = first_step + it
            bc1 = 1 - beta1 ** step
            bc2 = 1 - beta2 ** step
            rows[it] = (cur, cur / bc1, math.sqrt(bc2), 0.0)
        return rows.astype(np.float32)

    def run(self, niter, lr=0.01, schedule='cosine', lr_min=1e-6, reset_adam=True):
        """Runs `niter` fused iterations; returns the per-iteration losses as a CUDA tensor
        (no host sync inside — the reference syncs every iteration via float(loss), base_opt.py:366)."""
        if reset_adam or self.logd_m is None:
            self.reset_adam()
        if niter <= 0:
            return torch.zeros((0,), dtype=torch.float32, device=self.device)
        self.sched = torch.from_numpy(self.make_schedule(niter, lr, schedule, lr_min)).to(self.device)
        self.loss_out = torch.zeros((niter,), dtype=torch.float32, device=self.device)
        if self.shards is not None:
            with torch.cuda.device(self.device):
                self._sync_start()
                self.prepare()
                d = self._desc()
                for it in range(niter):
                    self._split_iteration(d, it)
                self._sync_end()
            return self.loss_out
        if not getattr(self, '_prepared', False):
            self.prepare()
        d = self._desc()
        _lib.launch(self.device, 'd3r_align_run', C.byref(d), 0, niter)
        return self.loss_out

    # ------------------------------------------------------------------ sharded iterations
    def _src(self, r):
        """Global rank of rank r of the engine's group."""
        return tdist.get_global_rank(self.group, r) if self.group is not None else r

    def _sync_start(self):
        """One broadcast of rank 0's log-depths and small parameters: every rank starts from the same parameters, whatever
        its own initialisation drew."""
        nl = self.logd.numel()
        buf = torch.cat((self.logd, self.small))
        tdist.broadcast(buf, src=self._src(0), group=self.group)
        self.logd.copy_(buf[:nl])
        self.small.copy_(buf[nl:])

    def _split_iteration(self, d, it):
        """Pixel pass over this rank's items, the exact integer all-reduce of the accumulators, the small step: all three on
        the engine's stream, nothing waits on the host."""
        if self.n_items:
            _lib.launch(self.device, 'd3r_align_pixel_pass', C.byref(d), it)
        tdist.all_reduce(self._reduce, op=tdist.ReduceOp.SUM, group=self.group)
        _lib.launch(self.device, 'd3r_align_small_step', C.byref(d), it)

    def _sync_end(self, flat=None):
        """Every owner broadcasts its images' slice of `flat` (default: the log-depths), laid out like `logd`, so that every
        rank holds the whole scene."""
        flat = self.logd if flat is None else flat
        for r, (a, b) in enumerate(self.shards):
            if b > a:
                tdist.broadcast(flat[int(self.pix_off[a]):int(self.pix_off[b])], src=self._src(r), group=self.group)

    def check_overflow(self):
        """Raises if a fixed-point accumulator left its range (host sync)."""
        flag = C.c_int32(0)
        d = self._desc()
        _lib.launch(self.device, 'd3r_align_overflow_flag', C.byref(d), C.byref(flag))
        if flag.value:
            raise _lib.D3RError('alignment: a gradient sum left the fixed-point accumulator range (partial >= 2^18 or total >= 2^22, or NaN / Inf); '
                                'rescale the scene (pointmaps are expected in metric-like units)')

    def evaluate_loss(self):
        """net.forward(): the objective at the current parameters, nothing updated."""
        self.sched = torch.zeros((1, 4), dtype=torch.float32, device=self.device)
        self.loss_out = torch.zeros((1,), dtype=torch.float32, device=self.device)
        if self.shards is not None:     # sharded: the objective at rank 0's parameters, the same value on every rank
            with torch.cuda.device(self.device):
                self._sync_start()
                self.prepare()
                self._split_iteration(self._desc(eval_only=True), 0)
            return self.loss_out[0]
        self.prepare()
        d = self._desc(eval_only=True)
        _lib.launch(self.device, 'd3r_align_run', C.byref(d), 0, 1)
        return self.loss_out[0]

    def loss_and_grad(self, entry_loss=False):
        """net.forward() + loss.backward() at the current parameters in one launch (d3r_align_loss_grad); nothing is
        updated.  Returns (loss, logd_grad, small_grad, entry_loss): a 0-dim loss, dL/dlog-depth laid out like `logd`
        (0 on padding pixels), dL/d(raw parameter) in the `small` layout (split it with split_small) and, when asked
        for, the (E, 2) coefficient-weighted loss of every (edge, side), else None.  Every tensor is freshly allocated,
        so results of two calls never alias."""
        if self.shards is not None:
            raise NotImplementedError('loss_and_grad is the single-GPU launch; a sharded engine takes the objective and its '
                                      'gradient with sharded_loss_and_grad, which every rank of the group calls')
        dev = self.device
        loss = torch.zeros((), dtype=torch.float32, device=dev)
        logd_grad = torch.zeros_like(self.logd)
        small_grad = torch.empty((self.n_small,), dtype=torch.float32, device=dev)
        ent = torch.empty((self.E, 2), dtype=torch.float32, device=dev) if entry_loss else None
        self.prepare()
        d = self._desc()
        d.loss_out = loss.data_ptr()
        _lib.launch(self.device, 'd3r_align_loss_grad', C.byref(d), logd_grad.data_ptr(), small_grad.data_ptr(),
                    ent.data_ptr() if ent is not None else None)
        return loss, logd_grad, small_grad, ent

    def sharded_loss_and_grad(self, entry_loss=False):
        """loss_and_grad of a sharded engine, and like run() a collective: every rank of the group calls it.  The objective
        is taken at rank 0's parameters (one broadcast, as evaluate_loss does).  This rank's gradient pixel pass
        (d3r_align_grad_pixel_pass) writes the log-depth gradients of its own images, one all-reduce combines the accumulator
        block, every rank's gradient small step (d3r_align_grad_small_step) forms the same loss, small-parameter gradients
        and entry losses, and one broadcast per owner of its images' log-depth gradients gives every rank all of them.
        Returns what loss_and_grad returns, bit-identical on every rank; on a one-rank group the bits of loss_and_grad."""
        if self.shards is None:
            raise ValueError('sharded_loss_and_grad needs a sharded engine (shards=); use loss_and_grad')
        dev = self.device
        loss = torch.zeros((), dtype=torch.float32, device=dev)
        logd_grad = torch.zeros_like(self.logd)
        small_grad = torch.empty((self.n_small,), dtype=torch.float32, device=dev)
        ent = torch.empty((self.E, 2), dtype=torch.float32, device=dev) if entry_loss else None
        with torch.cuda.device(dev):
            self._sync_start()
            self.prepare()
            d = self._desc()
            d.loss_out = loss.data_ptr()
            if self.n_items:
                _lib.launch(dev, 'd3r_align_grad_pixel_pass', C.byref(d), logd_grad.data_ptr())
            tdist.all_reduce(self._reduce, op=tdist.ReduceOp.SUM, group=self.group)
            _lib.launch(dev, 'd3r_align_grad_small_step', C.byref(d), small_grad.data_ptr(), ent.data_ptr() if ent is not None else None)
            # owner ranges are broadcast, not summed: an all-reduce over zero-filled ranges would turn -0.0 into +0.0
            self._sync_end(logd_grad)
        return loss, logd_grad, small_grad, ent

    def pts3d(self):
        """(sum stride_i, 3) world points of every image's pixels."""
        self.prepare()
        out = torch.zeros((int(self.pix_off[-1]), 3), dtype=torch.float32, device=self.device)
        d = self._desc()
        _lib.launch(self.device, 'd3r_align_pts3d', C.byref(d), out.data_ptr())
        return out
