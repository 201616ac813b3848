"""inference(): batched pairwise forward (API mirror of dust3r/inference.py:14-78).

Same contract as the reference: takes the `make_pairs` list, returns {'view1','view2','pred1','pred2','loss'}
with every tensor ON CPU, concatenated over pairs in input order (lists when image sizes are mixed).
Differences are internal: the list runs as C-ABI encode and decode calls (model.encode_images / model.decode_pairs:
d3r_encode_images, d3r_decode_pairs) that encode each distinct image once and decode pairs from those features, in
batches of one (size, size) group each when sizes are mixed; device->host copies of the predictions go through pinned
buffers and overlap the next calls' compute, and `keep_on_device=True` (extension) skips the host round trip for callers
that feed global_aligner next (SURVEY §8f rank 2)."""
from __future__ import annotations

import os

import torch
import tqdm

from .utils.device import to_cpu, collate_with_cat
from .utils.geometry import geotrf


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


def get_pred_pts3d(gt, pred, use_pose=False):
    """inference.py:81-103: the predicted points of a view -- pred['pts3d'] (moved by pred['camera_pose'] when use_pose), or
    pred['pts3d_in_other_view'] as it is (use_pose must then be set).  DUSt3R's heads never predict the depth / pseudo-focal
    pair the reference also accepts, so that form raises."""
    if 'depth' in pred and 'pseudo_focal' in pred:
        raise NotImplementedError('predictions given as depth + pseudo_focal are not supported: DUSt3R heads return pts3d')
    if 'pts3d' in pred:
        pts3d = pred['pts3d']
    elif 'pts3d_in_other_view' in pred:
        assert use_pose is True
        return pred['pts3d_in_other_view']
    else:
        raise KeyError('the prediction has neither pts3d nor pts3d_in_other_view')
    if use_pose:
        camera_pose = pred.get('camera_pose')
        assert camera_pose is not None
        pts3d = geotrf(camera_pose, pts3d)
    return pts3d


def loss_of_one_batch(batch, model, criterion, device, symmetrize_batch=False, use_amp=False, ret=None):
    """inference.py:32-52: moves the batch to `device`, optionally symmetrises it, runs the model and, when a criterion is
    given (dust3r_b200.losses), evaluates criterion(view1, view2, pred1, pred2) -> (loss, details) on the predictions.
    `use_amp` is accepted for the reference's signature; the forward's precision is fixed by the model."""
    view1, view2 = batch
    for view in batch:
        for name in view.keys():
            if name in _IGNORE:
                continue
            view[name] = view[name].to(device, non_blocking=True)
    if symmetrize_batch:
        view1, view2 = make_batch_symmetric(batch)
    pred1, pred2 = model(view1, view2)
    loss = criterion(view1, view2, pred1, pred2) if criterion is not None else None
    result = dict(view1=view1, view2=view2, pred1=pred1, pred2=pred2, loss=loss)
    return result[ret] if ret else result


def check_if_same_size(pairs):
    shapes1 = [img1['img'].shape[-2:] for img1, img2 in pairs]
    shapes2 = [img2['img'].shape[-2:] for img1, img2 in pairs]
    return all(shapes1[0] == s for s in shapes1) and all(shapes2[0] == s for s in shapes2)


_POOL = None


def _copy_pool():
    global _POOL
    if _POOL is None:
        from concurrent.futures import ThreadPoolExecutor
        _POOL = ThreadPoolExecutor(max_workers=max(1, min(8, (os.cpu_count() or 2) // 2)))
    return _POOL


def _fill_pinned(jobs, wait=True):
    """Run each (pinned destination, source) copy of `jobs` on a small thread pool (Tensor.copy_ releases the GIL, one
    thread saturates only ~10 GB/s of host bandwidth).  With wait=False the copies are left running in the background and
    their futures returned."""
    futs = [_copy_pool().submit(d.copy_, t) for d, t in jobs]
    if not wait:
        return futs
    for f in futs:
        f.result()
    return []


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


def _distinct_images(rows):
    """The distinct images of the rows of both views, by storage identity (make_pairs reuses one view dict per image in
    many pairs), in order of first use; the (view, row) of each one's first use; per view the index of each row's image."""
    uniq, first, gidx = {}, [], ([], [])
    for k in range(2):
        for i, t in enumerate(rows[k]):
            key = (t.data_ptr(), tuple(t.shape), tuple(t.stride()))
            if key not in uniq:
                uniq[key] = len(first)
                first.append((k, i))
            gidx[k].append(uniq[key])
    return [rows[k][i] for k, i in first], first, gidx


def _groups(gidx, mb):
    """Rows of the pipeline's groups: the list is cut into the shortest runs of consecutive rows that share no image with
    another run, and consecutive runs are joined while the group stays within `mb` rows (a longer run is a group alone)."""
    last = [0] * (1 + max(max(ix) for ix in gidx))
    for ix in gidx:
        for i, j in enumerate(ix):
            last[j] = max(last[j], i)
    groups, start, end = [], 0, 0
    for i in range(len(gidx[0])):
        end = max(end, last[gidx[0][i]], last[gidx[1][i]])
        if i == end:
            if groups and i + 1 - groups[-1].start <= mb:
                groups[-1] = range(groups[-1].start, i + 1)
            else:
                groups.append(range(start, i + 1))
            start = i + 1
    return groups


def _takes_pipeline(pairs, model, dev):
    """Whether inference() runs `pairs` as encode / decode calls.  The rest -- ManyAR batches of a landscape_only model,
    a true_shape other than its tensor's size, view dicts of several images in a list of several sizes, CPU stand-ins and
    models without encode_images / decode_pairs -- runs the reference's loop, where forward() checks and handles it."""
    if dev.type != 'cuda' or not (hasattr(model, 'encode_images') and hasattr(model, 'decode_pairs')) or not pairs:
        return False
    views = {id(v): v for pair in pairs for v in pair}.values()
    for v in views:
        hw = tuple(int(s) for s in v['img'].shape[-2:])
        ts = v.get('true_shape')
        if ts is not None and any(tuple(s) != hw for s in torch.as_tensor(ts).reshape(-1, 2).tolist()):
            return False
        if getattr(model, 'landscape_only', True) and hw[0] > hw[1]:
            return False
    return check_if_same_size(pairs) or all(int(v['img'].shape[0]) == 1 for v in views)


def _pipeline(pairs, model, dev, mb, verbose, keep_on_device, return_images):
    """inference() as encode / decode calls, group by group (_groups): the group's distinct images are uploaded on a copy
    stream and encoded once, one size at a time, in calls of at most 2 * mb images (what forward() on mb pairs encodes);
    its pairs are decoded per (view-1 size, view-2 size) in input order, at most mb per call, and the predictions copied out
    on a second side stream -- so the upload of the next group and the download of the last overlap the compute."""
    rows = ([], [])   # one (1,3,H,W) image per row: a view dict of k images is k pairs
    for a, b in pairs:
        k = int(a['img'].shape[0])
        assert int(b['img'].shape[0]) == k, 'both views of a pair must hold the same number of images'
        for r, v in zip(rows, (a, b)):
            r.extend([v['img']] if k == 1 else v['img'].split(1))
    n = len(rows[0])
    single = check_if_same_size(pairs)
    order, first, gidx = _distinct_images(rows)
    # An image that is neither pinned nor on the GPU goes up from a pinned copy: with one size and images returned, its first
    # row in the returned views (the other rows are filled in the background, call by call); with several sizes and host
    # images returned, a pinned copy kept for the returned views; otherwise a staging buffer of one encode call's images.
    img_pin = [torch.empty((n,) + tuple(r[0].shape[1:]), dtype=r[0].dtype, pin_memory=True) for r in rows] \
        if single and return_images else None
    keep_host = return_images and not single and not keep_on_device
    returned = {}   # several sizes, images returned: image -> its pinned (or, keep_on_device, device) copy
    main = torch.cuda.current_stream(dev)
    up, side = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
    up.wait_stream(main)   # images written on the device before the call
    outs, preds, pending = None, [None] * n, []
    with tqdm.tqdm(total=n, disable=not verbose) as bar:
        for g in _groups(gidx, mb):
            js = sorted({ix[i] for ix in gidx for i in g})
            src = {}   # image -> the pinned copy it is uploaded from
            if img_pin is not None:
                src = {j: img_pin[k][i:i + 1] for j in js if not _uploadable(order[j], dev) for k, i in [first[j]]}
                _fill_pinned([(src[j], order[j]) for j in src])
                filled = {first[j] for j in src}
            by_size, feats, at = {}, {}, {}   # at: image -> (its size, its row in that size's features)
            for j in js:
                by_size.setdefault(tuple(order[j].shape[-2:]), []).append(j)
            for hw, sj in by_size.items():
                parts = []
                for c in range(0, len(sj), 2 * mb):
                    chunk = sj[c:c + 2 * mb]
                    shape, dtype = (len(chunk),) + tuple(order[chunk[0]].shape[1:]), order[chunk[0]].dtype
                    staged = [j for j in chunk if j not in src and (keep_host or not _uploadable(order[j], dev))]
                    if staged:
                        stage = torch.empty((len(staged),) + shape[1:], dtype=dtype, pin_memory=True)
                        src.update((j, stage[r:r + 1]) for r, j in enumerate(staged))
                        _fill_pinned([(src[j], order[j]) for j in staged])
                    # allocated on the copy stream and recorded on the main one: the memory is reused once the encode
                    # that reads it has run, without making the next upload wait for this group's compute
                    with torch.cuda.stream(up):
                        img = torch.empty(shape, dtype=dtype, device=dev)
                        for r, j in enumerate(chunk):
                            img[r:r + 1].copy_(src.get(j, order[j]), non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(up)
                    main.wait_event(ev)
                    img.record_stream(main)
                    parts.append(model.encode_images(img))
                    if return_images and not single:
                        returned.update((j, img[r:r + 1] if keep_on_device else src[j]) for r, j in enumerate(chunk))
                feats[hw] = parts[0] if len(parts) == 1 else torch.cat(parts)
                at.update((j, (hw, r)) for r, j in enumerate(sj))
            calls = {}
            for i in g:
                calls.setdefault((at[gidx[0][i]][0], at[gidx[1][i]][0]), []).append(i)
            for (hw1, hw2), members in calls.items():
                for c in range(0, len(members), mb):
                    sel = members[c:c + mb]
                    if img_pin is not None:
                        pending += _fill_pinned([(img_pin[k][i:i + 1], rows[k][i]) for k in range(2) for i in sel
                                                 if (k, i) not in filled], wait=False)
                    pred1, pred2 = model.decode_pairs(feats[hw1], [at[gidx[0][i]][1] for i in sel],
                                                      feats[hw2], [at[gidx[1][i]][1] for i in sel])
                    flat = {('pred1', key): t for key, t in pred1.items()}
                    flat.update({('pred2', key): t for key, t in pred2.items()})
                    if single:   # one stacked result; a group's rows are consecutive
                        if outs is None:
                            outs = {key: torch.empty((n,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev if keep_on_device else None,
                                                     pin_memory=not keep_on_device) for key, t in flat.items()}
                        dst = {key: outs[key][sel[0]:sel[0] + len(sel)] for key in flat}
                    elif keep_on_device:
                        dst = flat
                    else:
                        dst = {key: torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for key, t in flat.items()}
                    if dst is not flat:
                        ev = torch.cuda.Event()
                        ev.record(main)
                        side.wait_event(ev)
                        with torch.cuda.stream(side):
                            for key, t in flat.items():
                                dst[key].copy_(t, non_blocking=True)
                                t.record_stream(side)
                    if not single:
                        for r, i in enumerate(sel):
                            preds[i] = tuple({key: t[r:r + 1] for (w, key), t in dst.items() if w == which}
                                             for which in ('pred1', 'pred2'))
                    bar.update(len(sel))
            del feats
    side.synchronize()
    for f in pending:
        f.result()
    views = ([a for a, b in pairs], [b for a, b in pairs])
    if single:
        vs = [{key: collate_with_cat([v[key] for v in views[k]]) for key in views[k][0] if key != 'img'} for k in range(2)]
        if return_images:
            for k in range(2):
                vs[k]['img'] = img_pin[k]
        res = dict(view1=vs[0], view2=vs[1], pred1={}, pred2={}, loss=None)
        for (which, key), t in outs.items():
            res[which][key] = t
        return res
    # several sizes: the reference's one-pair-per-call loop (inference.py:60-72), lists with one entry per pair
    results = []
    for i in range(n):
        vs = []
        for k in range(2):
            v = collate_with_cat([views[k][i]])
            if return_images:
                v['img'] = returned[gidx[k][i]]
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
    keep_on_device; lists with one entry per pair when the image sizes are mixed.  return_images=False (extension) leaves
    'img' out of the returned views and skips the host copy behind them where the upload does not need it.

    On a CUDA device, a model with encode_images / decode_pairs runs every list _takes_pipeline accepts as one pipeline
    (_pipeline): each distinct image of the list (by storage: make_pairs shares one view dict between many pairs) is
    uploaded and encoded once, and its pairs are decoded from those features in calls of at most one micro-batch
    (_micro_batch), overlapped with the upload of the next images and the download of the last predictions.  Every other
    list runs the reference's loop of forward() calls."""
    if verbose:
        print(f'>> Inference with model on {len(pairs)} image pairs')
    dev = torch.device(device)
    if _takes_pipeline(pairs, model, dev):
        return _pipeline(pairs, model, dev, _micro_batch(batch_size), verbose, keep_on_device, return_images)
    multiple_shapes = not check_if_same_size(pairs)
    result = []
    bs = 1 if multiple_shapes else batch_size
    for i in tqdm.trange(0, len(pairs), bs, disable=not verbose):
        res = loss_of_one_batch(collate_with_cat(pairs[i:i + bs]), model, None, device)
        result.append(res if keep_on_device else to_cpu(res))
    return collate_with_cat(result, lists=multiple_shapes)
