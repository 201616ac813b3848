"""inference(): batched pairwise forward (API mirror of dust3r/inference.py:14-78).

Same contract as the reference: takes the `make_pairs` list, returns {'view1','view2','pred1','pred2','loss'}
with every tensor ON CPU, concatenated over pairs in input order (lists when image sizes are mixed).
Differences are internal: each batch runs as C-ABI encode and decode calls (d3r_encode_images, d3r_decode_pairs),
device->host copies of the predictions go through pinned staging buffers and overlap the next batch's compute, and
`keep_on_device=True` (extension) skips the host round trip for callers that feed global_aligner next
(SURVEY §8f rank 2).  Pair lists that share images (make_pairs) encode each image once (model.encode_images) and
decode every batch from those features (model.decode_pairs); pair lists of several image sizes are decoded in
batches of one (size, size) group each instead of one pair per call."""
from __future__ import annotations

import os

import torch
import tqdm

from .utils.device import to_cpu, collate_with_cat


def _interleave_imgs(img1, img2):
    res = {}
    for key, value1 in img1.items():
        value2 = img2[key]
        if isinstance(value1, torch.Tensor):
            value = torch.stack((value1, value2), dim=1).flatten(0, 1)
        else:
            value = [x for pair in zip(value1, value2) for x in pair]
        res[key] = value
    return res


def make_batch_symmetric(batch):
    view1, view2 = batch
    return _interleave_imgs(view1, view2), _interleave_imgs(view2, view1)


_IGNORE = {'depthmap', 'dataset', 'label', 'instance', 'idx', 'true_shape', 'rng'}


def loss_of_one_batch(batch, model, criterion, device, symmetrize_batch=False, use_amp=False, ret=None):
    """inference.py:32-52.  `criterion` must be None (training losses are outside the hot paths)."""
    view1, view2 = batch
    for view in batch:
        for name in view.keys():
            if name in _IGNORE:
                continue
            view[name] = view[name].to(device, non_blocking=True)
    if symmetrize_batch:
        view1, view2 = make_batch_symmetric(batch)
    if criterion is not None:
        raise NotImplementedError('training criteria are not part of the inference hot path')
    pred1, pred2 = model(view1, view2)
    result = dict(view1=view1, view2=view2, pred1=pred1, pred2=pred2, loss=None)
    return result[ret] if ret else result


def check_if_same_size(pairs):
    shapes1 = [img1['img'].shape[-2:] for img1, img2 in pairs]
    shapes2 = [img2['img'].shape[-2:] for img1, img2 in pairs]
    return all(shapes1[0] == s for s in shapes1) and all(shapes2[0] == s for s in shapes2)


_POOL = None
_TRACE = None   # set to a list to collect (label, perf_counter) host timestamps of the pipeline (diagnostics)


def _mark(label):
    if _TRACE is not None:
        import time
        _TRACE.append((label, time.perf_counter()))


def _copy_pool():
    global _POOL
    if _POOL is None:
        from concurrent.futures import ThreadPoolExecutor
        _POOL = ThreadPoolExecutor(max_workers=max(1, min(8, (os.cpu_count() or 2) // 2)))
    return _POOL


def _fill_pinned(dst, tensors, row0, wait=True):
    """Copy each view's image rows into the pinned staging tensor `dst` starting at row `row0` (memcpy on a small
    thread pool: Tensor.copy_ releases the GIL, one thread saturates only ~10 GB/s of host bandwidth).
    Returns (next row, futures); with wait=False the copies are left running in the background."""
    jobs, r = [], row0
    for t in tensors:
        k = int(t.shape[0])
        jobs.append((dst[r:r + k], t))
        r += k
    futs = [_copy_pool().submit(d.copy_, t) for d, t in jobs]
    if wait:
        for f in futs:
            f.result()
        futs = []
    return r, futs


def _uploadable(t, dev):
    """Sources the copy stream can read directly: pinned host memory, or an image that already lives on the target GPU
    (load_images(..., device=...): resized and normalised there)."""
    if not t.is_cuda:
        return t.is_pinned()
    return t.device.index == (dev.index if dev.index is not None else torch.cuda.current_device())


def _micro_batch(batch_size):
    """Pairs per forward call.  A user batch of >= 16 pairs is run as two halves so that the host-side
    staging + H2D of one half and the D2H of the other overlap the GPU compute (per-pair results do not depend on
    the batch they are computed in); halves stay even so symmetrised (a,b),(b,a) neighbours are kept together."""
    if batch_size < 16:
        return batch_size
    half = (batch_size + 1) // 2
    return half + (half & 1)


def _distinct_images(views):
    """The distinct image tensors of single-image view dicts, by identity (make_pairs reuses one dict per image in many
    pairs), in order of first use, and per view the index of each pair's image in that list."""
    uniq, order, gidx = {}, [], ([], [])
    for k in range(2):
        for v in views[k]:
            t = v['img']
            key = (t.data_ptr(), tuple(t.shape), tuple(t.stride()))
            if key not in uniq:
                uniq[key] = len(order)
                order.append(t)
            gidx[k].append(uniq[key])
    return order, gidx


def _upload(ts, dev, up):
    """One device tensor holding the images `ts` (each (1,3,H,W), one size), copied on the stream `up`; the current stream
    waits for the copy."""
    main = torch.cuda.current_stream(dev)
    out = torch.empty((len(ts),) + tuple(ts[0].shape[1:]), dtype=ts[0].dtype, device=dev)
    up.wait_stream(main)
    with torch.cuda.stream(up):
        if all(_uploadable(t, dev) for t in ts):
            for j, t in enumerate(ts):
                out[j:j + 1].copy_(t, non_blocking=True)
        else:
            stage = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
            _fill_pinned(stage, ts, 0, wait=True)
            out.copy_(stage, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record(up)
    main.wait_event(ev)
    return out


def _encode(model, imgs, chunk):
    """Encoder features of every image of `imgs`, in calls of at most `chunk` images (what bounds the encoder's workspace:
    forward() on `chunk // 2` pairs encodes up to `chunk` images)."""
    parts = [model.encode_images(imgs[c:c + chunk]) for c in range(0, int(imgs.shape[0]), chunk)]
    return parts[0] if len(parts) == 1 else torch.cat(parts)


def _inference_mixed(pairs, model, dev, batch_size, verbose, keep_on_device, return_images):
    """Pair lists of more than one image size (one image per view dict, a model with landscape_only=False): every distinct
    image is uploaded and encoded once, one size at a time, and the pairs of each (view-1 size, view-2 size) group are
    decoded in input order, `batch_size` pairs per call.  The result is the reference's one-pair-per-call loop
    (inference.py:60-72): lists with one entry per pair, in input order, with the same values -- a pair's output does not
    depend on the batch it is computed in."""
    n = len(pairs)
    views = ([a for a, b in pairs], [b for a, b in pairs])
    order, gidx = _distinct_images(views)
    by_size = {}
    for j, t in enumerate(order):
        by_size.setdefault(tuple(t.shape[-2:]), []).append(j)
    slot = [None] * len(order)   # distinct image -> (its size, its row in that size's feature tensor)
    up = torch.cuda.Stream(device=dev)
    imgs, feats = {}, {}
    for hw, js in by_size.items():
        for r, j in enumerate(js):
            slot[j] = (hw, r)
        imgs[hw] = _upload([order[j] for j in js], dev, up)
        feats[hw] = _encode(model, imgs[hw], 2 * batch_size)
        if not return_images:
            del imgs[hw]
        elif not keep_on_device:
            imgs[hw] = imgs[hw].cpu()
    groups = {}
    for i in range(n):
        groups.setdefault((slot[gidx[0][i]][0], slot[gidx[1][i]][0]), []).append(i)
    preds = [None] * n
    with tqdm.tqdm(total=n, disable=not verbose) as bar:
        for (hw1, hw2), members in groups.items():
            for c in range(0, len(members), batch_size):
                sel = members[c:c + batch_size]
                out = model.decode_pairs(feats[hw1], [slot[gidx[0][i]][1] for i in sel],
                                         feats[hw2], [slot[gidx[1][i]][1] for i in sel])
                out = out if keep_on_device else to_cpu(out)
                for j, i in enumerate(sel):
                    preds[i] = tuple({key: t[j:j + 1] for key, t in p.items()} for p in out)
                bar.update(len(sel))
    results = []
    for i in range(n):
        vs = []
        for k in range(2):
            v = collate_with_cat([views[k][i]])
            if return_images:
                hw, r = slot[gidx[k][i]]
                v['img'] = imgs[hw][r:r + 1]
            else:
                del v['img']
            if keep_on_device:   # where loss_of_one_batch puts the other fields of a view
                v.update({key: t.to(dev, non_blocking=True) for key, t in v.items()
                          if key != 'img' and key not in _IGNORE and torch.is_tensor(t)})
            vs.append(v)
        results.append(dict(view1=vs[0], view2=vs[1], pred1=preds[i][0], pred2=preds[i][1], loss=None))
    return collate_with_cat(results, lists=True)


@torch.no_grad()
def inference(pairs, model, device, batch_size=8, verbose=True, keep_on_device=False, return_images=True):
    """inference.py:55-72.  Returns {'view1','view2','pred1','pred2','loss'}; tensors on CPU (pinned) unless
    keep_on_device.  Software pipeline over micro-batches: images are gathered into pinned host memory (which is
    also the returned, collated view; return_images=False -- extension -- leaves 'img' out of the returned views and skips
    that copy where the upload does not need it), uploaded on a copy stream, run through one forward call, and the
    predictions are copied D2H on a second side stream into the final (whole pair list) pinned output -- the
    upload of batch k+1 and the download of batch k-1 overlap the compute of batch k."""
    if verbose:
        print(f'>> Inference with model on {len(pairs)} image pairs')
    multiple_shapes = not check_if_same_size(pairs)
    dev = torch.device(device)
    if (multiple_shapes and dev.type == 'cuda' and hasattr(model, 'decode_pairs') and not getattr(model, 'landscape_only', True)
            and all(int(v['img'].shape[0]) == 1 for pair in pairs for v in pair)):
        return _inference_mixed(pairs, model, dev, batch_size, verbose, keep_on_device, return_images)
    fused = dev.type == 'cuda' and not multiple_shapes and len(pairs) > 0
    if not fused:
        # mixed image sizes (batch size forced to 1, lists instead of stacked tensors) or non-CUDA stand-in
        # models used by host-side tests: plain reference control flow
        result = []
        bs = 1 if multiple_shapes else batch_size
        for i in tqdm.trange(0, len(pairs), bs, disable=not verbose):
            res = loss_of_one_batch(collate_with_cat(pairs[i:i + bs]), model, None, device)
            result.append(res if keep_on_device else to_cpu(res))
        return collate_with_cat(result, lists=multiple_shapes)

    _mark('begin')
    n = len(pairs)
    views = ([a for a, b in pairs], [b for a, b in pairs])
    rows = [sum(int(v['img'].shape[0]) for v in vs) for vs in views]
    assert rows[0] == rows[1], 'both views of a pair must hold the same number of images'
    proto = [vs[0]['img'] for vs in views]
    # pinned staging = the collated 'img' of the returned views; device copies of the whole pair list (a few MB / pair)
    img_pin = None    # allocated below, unless the caller does not want the images back and the upload does not stage through it
    img_dev = None    # device copies of both views: only the path without shared images needs them (allocated there)
    meta_all = [{key: collate_with_cat([v[key] for v in vs]) for key in vs[0] if key != 'img'} for vs in views]
    _mark('alloc+meta')
    outs = None
    main = torch.cuda.current_stream(dev)
    up, side = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
    up.wait_stream(main)
    mb = _micro_batch(batch_size)
    r0 = 0
    pending = []
    # pair lists from make_pairs reuse the same image dict in many pairs (n images -> up to n(n-1) pairs): upload and encode
    # every distinct image once, then decode each micro-batch from those features through index maps -- the encoder runs
    # once per image of the list instead of twice per pair (its output for an image does not depend on what else is in
    # the batch, so results are unchanged).  Encoder calls take at most 2 * mb images, as forward() on mb pairs does.
    feats, gidx = None, ([], [])
    if hasattr(model, 'decode_pairs') and all(int(v['img'].shape[0]) == 1 for vs in views for v in vs):
        order, gidx = _distinct_images(views)
        if len(order) < 2 * n:
            feats = _encode(model, _upload(order, dev, up), 2 * mb)
    all_pinned = all(_uploadable(v['img'], dev) for vs in views for v in vs)
    if return_images or not (feats is not None or all_pinned):
        img_pin = [torch.empty((rows[k],) + tuple(proto[k].shape[1:]), dtype=proto[k].dtype, pin_memory=True) for k in range(2)]
    for i in tqdm.trange(0, n, mb, disable=not verbose):
        chunk = (views[0][i:i + mb], views[1][i:i + mb])
        r1 = r0
        srcs = [[v['img'] for v in chunk[k]] for k in range(2)]
        direct = all(_uploadable(t, dev) for ts in srcs for t in ts)
        indexed = feats is not None
        for k in range(2):
            # sources already in pinned memory are uploaded straight from where they are; the collated copy that the
            # caller gets back is then filled in the background, off the critical path
            if img_pin is None:
                r1 = r0 + sum(int(t.shape[0]) for t in srcs[k])
                continue
            r1, futs = _fill_pinned(img_pin[k], srcs[k], r0, wait=not (direct or indexed))
            pending.extend(futs)
        _mark('fill')
        if indexed:
            _mark('h2d+meta')
            pred1, pred2 = model.decode_pairs(feats, gidx[0][i:i + mb], feats, gidx[1][i:i + mb])
        else:
            # device staging: two micro-batch sized buffers per view, used alternately (the reference holds one batch on the
            # GPU at a time; a whole-pair-list copy would grow by 4.7 MB per pair at 512x384).  A buffer is reused two
            # micro-batches later: the upload stream first waits for the forward that last read it.
            if img_dev is None:
                per_item = [int(v['img'].shape[0]) for v in views[0]]
                cap = max(sum(per_item[c:c + mb]) for c in range(0, n, mb))
                img_dev = [[torch.empty((cap,) + tuple(proto[k].shape[1:]), dtype=proto[k].dtype, device=dev) for k in range(2)]
                           for _ in range(2)]
                dev_free = [None, None]
            slot = (i // mb) & 1
            nrow = r1 - r0
            with torch.cuda.stream(up):
                if dev_free[slot] is not None:
                    up.wait_event(dev_free[slot])
                for k in range(2):
                    if direct:
                        r = 0
                        for t in srcs[k]:
                            img_dev[slot][k][r:r + int(t.shape[0])].copy_(t, non_blocking=True)
                            r += int(t.shape[0])
                    else:
                        img_dev[slot][k][:nrow].copy_(img_pin[k][r0:r1], non_blocking=True)
            ev_up = torch.cuda.Event()
            ev_up.record(up)
            main.wait_event(ev_up)
            d = [dict({key: collate_with_cat([v[key] for v in chunk[k]]) for key in chunk[k][0] if key != 'img'},
                      img=img_dev[slot][k][:nrow]) for k in range(2)]
            _mark('h2d+meta')
            pred1, pred2 = model(d[0], d[1])
            dev_free[slot] = torch.cuda.Event()
            dev_free[slot].record(main)
        _mark('forward-enqueued')
        flat = {('pred1', k): v for k, v in pred1.items()}
        flat.update({('pred2', k): v for k, v in pred2.items()})
        if outs is None:
            if keep_on_device:
                outs = {key: torch.empty((rows[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=dev) for key, t in flat.items()}
            else:
                outs = {key: torch.empty((rows[0],) + tuple(t.shape[1:]), dtype=t.dtype, pin_memory=True) for key, t in flat.items()}
        ev = torch.cuda.Event()
        ev.record(main)
        with torch.cuda.stream(side):
            side.wait_event(ev)
            for key, t in flat.items():
                outs[key][r0:r1].copy_(t, non_blocking=True)
                t.record_stream(side)
        _mark('d2h-enqueued')
        r0 = r1
    side.synchronize()
    for f in pending:
        f.result()
    _mark('synced')
    main.wait_stream(up)
    if return_images:
        res = dict(view1=dict(meta_all[0], img=img_pin[0]), view2=dict(meta_all[1], img=img_pin[1]), pred1={}, pred2={}, loss=None)
    else:
        res = dict(view1=dict(meta_all[0]), view2=dict(meta_all[1]), pred1={}, pred2={}, loss=None)
    for (which, k), t in outs.items():
        res[which][k] = t
    return res
