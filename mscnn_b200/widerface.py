"""The WIDER FACE drivers over the library: examples/widerface/run_mscnn_detection.m and run_cascademscnn.m run every
image at its own net input size (`imgW = 0; imgH = 0; max_size = 3072`, :34 / :55): the original size rounded to
multiples of 32, the longer side capped at 3072 (:70-81).  Here the images are grouped by that size and each group runs
as ordinary batches of one shape; the net's input shape changes only between batches.  Every image's detections are
those of the drivers' one-image-at-a-time loop, bit for bit.

    dets = widerface.run(net, frames, names)                 # {name: [k][5] = x y w h prob}, input order
    dets = widerface.run(drivers.make_nets(proto, weights, [0, 0]), frames, names)     # the same, on two nets
    widerface.write_results("detections/<comp_id>/<event>", dets)
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi

MAX_SIZE = 3072                 # run_mscnn_detection.m:34, run_cascademscnn.m:55
# Net-input pixels one batch may hold: 8 images of 768 x 2560 take about 25 GB of device memory.  A group of large
# images is cut into smaller batches (a 3072 x 3072 image runs alone); an image above the budget still runs, alone.
PIXEL_BUDGET = 8 * 768 * 2560


def plan_batches(org_hw, img_hw=(0, 0), max_size: int = MAX_SIZE, max_batch: int = 8,
                 pixel_budget: int = PIXEL_BUDGET) -> list[tuple[tuple[int, int], list[int]]]:
    """Batches for images of original sizes org_hw [(h, w)]: [((net_h, net_w), [image indices])].

    An image's net size is ops.widerface_net_size(h, w, *img_hw, max_size).  Images of one net size share batches of
    at most min(max_batch, pixel_budget // (net_h * net_w)) images, in input order.  Groups run from the largest net
    size down, so that the net's buffers reach their largest size with the first batch instead of growing batch after
    batch.  The result depends on the arguments alone, and every index appears exactly once."""
    from . import ops
    if max_batch < 1 or pixel_budget < 1:
        raise ValueError(f"max_batch ({max_batch}) and pixel_budget ({pixel_budget}) must be positive")
    groups: dict[tuple[int, int], list[int]] = {}
    for i, (h, w) in enumerate(org_hw):
        hw = ops.widerface_net_size(int(h), int(w), int(img_hw[0]), int(img_hw[1]), max_size)
        groups.setdefault(hw, []).append(i)
    batches = []
    for hw in sorted(groups, key=lambda s: (-s[0] * s[1], -s[0], -s[1])):
        per = max(1, min(max_batch, pixel_budget // (hw[0] * hw[1])))
        idx = groups[hw]
        batches += [(hw, idx[k:k + per]) for k in range(0, len(idx), per)]
    return batches


def run(nets, frames, names, cascade: bool = False, max_size: int = MAX_SIZE, max_batch: int = 8,
        pixel_budget: int = PIXEL_BUDGET, plans: dict | None = None, proposals: bool = False):
    """Final face detections of uint8 [h][w][3] host frames (any sizes) on `nets`, models.widerface nets (or, with
    cascade=True, models.widerface_cascade nets read at proposals_3rd / cls_prob_3rd_avg / output_bbox_3rd as
    run_cascademscnn.m:44-47 does), with the drivers' settings (net.widerface_detect_cfg).

    Returns {name: float32 [k][5] = x y w h prob} in input order: the kept rows of each image in the post-process's
    order, in original-image coordinates.  plans: a dict net size -> ops.Preprocess to reuse between calls (the plans
    keep the resize tables of every original size they have seen); new plans are added to it.

    nets: one net.Net, run on the calling thread and stream; or a list of nets (drivers.make_nets), each served by a
    host thread of its own (drivers.serve_batches, drivers.net_thread) taking plan_batches' batches, largest first,
    from one queue.  plans is then None or a list of one dict per net.  The result is the one-net result, bit for bit.

    proposals=True (plain nets only): returns (dets, props), props = {name: float64 [k][5] = x y w h score}, each
    image's proposal list at its own net size with proposal_thr -5 (run_mscnn_detection.m:55, :95-109)."""
    from . import drivers, net as mnet, ops
    names = list(names)
    if len(names) != len(frames) or len(set(names)) != len(names):
        raise ValueError("one distinct name per frame is needed")
    if cascade and proposals:
        raise ValueError("run_cascademscnn.m computes no proposal list")
    hw = ops.image_sizes(frames)
    kept: list[np.ndarray | None] = [None] * len(frames)
    props: list | None = [None] * len(frames) if proposals else None

    def result():
        dets = dict(zip(names, kept))
        return (dets, dict(zip(names, props))) if proposals else dets

    batches = plan_batches(hw, max_size=max_size, max_batch=max_batch, pixel_budget=pixel_budget)
    drivers.keep_readable(nets, ("proposals_3rd", "cls_prob_3rd_avg", "output_bbox_3rd") if cascade
                          else ("proposals_score", "cls_pred", "bbox_pred"))
    if not isinstance(nets, (list, tuple)):
        plans = {} if plans is None else plans
        for b in batches:
            _run_batch(nets, frames, hw, b, cascade, plans, kept, props)
        return result()
    if plans is None:
        plans = [{} for _ in nets]
    elif not isinstance(plans, (list, tuple)) or len(plans) != len(nets):
        raise ValueError("with several nets, plans is None or a list of one dict per net")
    per_net = dict(zip(map(id, nets), plans))
    precision = mnet.get_precision()

    def serve(net, take):
        with drivers.net_thread(net, precision):
            b = take()
            while b is not None:
                _run_batch(net, frames, hw, b, cascade, per_net[id(net)], kept, props)
                b = take()

    drivers.serve_batches(nets, batches, serve)
    return result()


def _run_batch(net, frames, hw, batch, cascade: bool, plans: dict, kept: list, props: list | None = None) -> None:
    """One plan_batches entry ((net_h, net_w), image indices) on `net` in the calling thread, into kept[i] (and
    props[i], props not None)."""
    import torch
    from . import drivers, net as mnet, ops
    (rz_h, rz_w), idx = batch
    n = len(idx)
    data = net.inputs[0]
    net.reshape_input(data, n, 3, rz_h, rz_w)
    pre = plans.get((rz_h, rz_w))
    if pre is None:
        pre = plans[(rz_h, rz_w)] = ops.Preprocess(tuple(hw[idx[0]]), (rz_h, rz_w))
    net.set_input_images(data, pre, [frames[i] for i in idx])
    net.forward_only()
    cfg, classes = mnet.widerface_detect_cfg(rz_h, rz_w)    # the original sizes come with the frames
    with torch.cuda.stream(mnet._net_stream()):
        dets = torch.empty((n, 1, cfg.max_rois_per_image, 5), dtype=torch.float32, device="cuda")
        counts = torch.empty((n, 1), dtype=torch.int32, device="cuda")
        if cascade:
            net.detect_cascade_classes(cfg, classes, dets.data_ptr(), counts.data_ptr(), stage="3rd",
                                       cls_prob="cls_prob_3rd_avg")
        else:
            net.detect_classes(cfg, classes, dets.data_ptr(), counts.data_ptr())
        if props is not None:
            pp = drivers.read_proposals(net, cfg, n)
        d, c = dets.cpu().numpy(), counts.cpu().numpy()
    for k, i in enumerate(idx):
        kept[i] = d[k, 0, :c[k, 0]].copy()
        if props is not None:
            props[i] = pp[k]


def write_results(event_dir, results) -> None:
    """<event_dir>/<name>.txt for every {name: [k][5] rows} of `results` (what run returns), as
    run_mscnn_detection.m:177-196 writes them: the name, the count, one "%d %d %d %d %f" row per detection (x y w h
    through MATLAB round, then the probability).  The directory and its missing parents are created."""
    names = list(results)
    rows = [np.asarray(results[k], dtype=np.float32).reshape(-1, 5) for k in names]
    counts = np.ascontiguousarray([len(r) for r in rows], dtype=np.int32)
    cap = max([1] + counts.tolist())
    dets = np.zeros((len(rows), cap, 5), dtype=np.float32)
    for i, r in enumerate(rows):
        dets[i, :len(r)] = r
    c_names = (C.c_char_p * max(len(names), 1))(*[k.encode() for k in names])
    capi.check(capi.lib().mscnn_widerface_write_results(str(event_dir).encode(), len(names), c_names, dets.ctypes.data,
                                                        counts.ctypes.data, cap), "widerface_write_results")
